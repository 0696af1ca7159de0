// fp32 CUDA-core implementation of DM_NeRF.forward (reference networks/dm_nerf.py:80-106), fused with the
// point generation + positional encoding of render.py:49-58 when called on rays.
//
// Role: the exact-fp32 path.  It serves (i) as the on-device cross-check for the tensor-core kernel,
// (ii) shapes the tensor-core kernel does not cover, (iii) DMNERF_IMPL_SIMT.  It keeps every activation
// on chip: one CTA owns a tile of 64 samples, the 256-wide hidden state lives in shared memory and each
// layer is computed in place from an 8x8 register tile per thread; weights stream from L2 in 16-deep
// K-slices that are transposed into shared memory.
#include "ray_ops.cuh"

namespace dmnerf {

namespace simt {
constexpr int TM = 64;      // samples per CTA
constexpr int NT = 256;     // threads per CTA
constexpr int KC = 16;      // K-slice staged per step
constexpr int LDE = 92;     // embedding buffer  [TM][90 (+2)]
constexpr int LDX = 324;    // main buffer       [TM][319 (+5)]   (324 % 32 == 4: rows land on distinct banks)
constexpr int LDB = 260;    // second buffer     [TM][256 (+4)]
constexpr size_t SMEM_BYTES = (size_t)(TM * LDE + TM * LDX + TM * LDB + KC * 256) * sizeof(float);

// Y[r][c] = act(b[c] + sum_k X[r][k] W[c][k]),  r < TM, c < N <= 256.  Y may alias X (results are held in
// registers until every thread has finished reading X).
template <bool RELU>
__device__ void layer(const float* Xs, int ldx, int K, const float* __restrict__ W, const float* __restrict__ bias,
                      int N, float* Ys, int ldy, float* Wt, float* __restrict__ Yg = nullptr, int rows_valid = 0) {
  const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.0f;

  for (int k0 = 0; k0 < K; k0 += KC) {
    const int kmax = min(KC, K - k0);
    __syncthreads();                                   // previous slice fully consumed
    {
      const int nrow = tid;                            // thread <-> output feature
      const float* wrow = W + (size_t)nrow * K + k0;
#pragma unroll
      for (int kk = 0; kk < KC; ++kk)
        Wt[kk * 256 + nrow] = (nrow < N && kk < kmax) ? __ldg(wrow + kk) : 0.0f;
    }
    __syncthreads();
#pragma unroll 4
    for (int kk = 0; kk < kmax; ++kk) {
      float xv[8], wv[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) xv[i] = Xs[(ty * 8 + i) * ldx + k0 + kk];
#pragma unroll
      for (int j = 0; j < 8; ++j) wv[j] = Wt[kk * 256 + tx + 32 * j];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(xv[i], wv[j], acc[i][j]);
    }
  }
  __syncthreads();                                     // all reads of Xs done: in-place write is safe
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = tx + 32 * j;
    if (c < N) {
      const float bv = __ldg(bias + c);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float v = acc[i][j] + bv;
        if (RELU) v = fmaxf(v, 0.0f);
        Ys[(ty * 8 + i) * ldy + c] = v;
        if (Yg != nullptr && ty * 8 + i < rows_valid) Yg[(size_t)(ty * 8 + i) * N + c] = v;   // training: keep the activation
      }
    }
  }
  __syncthreads();
}

// Narrow output heads (N small): one thread per (row, feature) dot product, written straight to global.
__device__ void head(const float* Xs, int ldx, int K, const float* __restrict__ W, const float* __restrict__ bias, int N,
                     float* __restrict__ out, int out_ld, int out_col, int rows_valid) {
  for (int idx = threadIdx.x; idx < TM * N; idx += NT) {
    const int r = idx / N, c = idx % N;
    if (r >= rows_valid) continue;
    const float* xr = Xs + r * ldx;
    const float* wr = W + (size_t)c * K;
    float a = 0.0f;
    for (int k = 0; k < K; ++k) a = fmaf(xr[k], __ldg(wr + k), a);
    out[(size_t)r * out_ld + out_col + c] = a + __ldg(bias + c);
  }
}

__global__ void __launch_bounds__(NT, 1)
mlp_simt_kernel(NetParams p, const float* __restrict__ x, const float* __restrict__ rays_o,
                const float* __restrict__ rays_d, const float* __restrict__ z, int64_t m, int S,
                float* __restrict__ out, float* __restrict__ acts) {
  extern __shared__ float smem[];
  float* E = smem;                      // [TM][LDE]  [emb_pos 63 | emb_dir 27]
  float* X = E + TM * LDE;              // [TM][LDX]
  float* B = X + TM * LDX;              // [TM][LDB]
  float* Wt = B + TM * LDB;             // [KC][256]
  const int tid = threadIdx.x;
  const int C = 4 + p.ins_num + 1;

  for (int64_t row0 = (int64_t)blockIdx.x * TM; row0 < m; row0 += (int64_t)gridDim.x * TM) {
    const int rows_valid = (int)min((int64_t)TM, m - row0);
    __syncthreads();
    // ---- inputs -> E
    if (x) {
      for (int idx = tid; idx < TM * CH_IN; idx += NT) {
        const int r = idx / CH_IN, c = idx % CH_IN;
        E[r * LDE + c] = (r < rows_valid) ? x[(row0 + r) * CH_IN + c] : 0.0f;
      }
    } else {
      constexpr int SLOTS = (L_POS + 1) + (L_DIR + 1);          // 11 position slots + 5 direction slots
      for (int idx = tid; idx < TM * SLOTS; idx += NT) {
        const int r = idx / SLOTS, sl = idx % SLOTS;
        float* e = E + r * LDE;
        if (r >= rows_valid) {
          if (sl == 0) for (int c = 0; c < CH_IN; ++c) e[c] = 0.0f;
          continue;
        }
        const int64_t row = row0 + r, ray = row / S;
        const float d[3] = {rays_d[ray * 3], rays_d[ray * 3 + 1], rays_d[ray * 3 + 2]};
        if (sl <= L_POS) {
          const float zz = z[row];
          float pt[3];
#pragma unroll
          for (int c = 0; c < 3; ++c) pt[c] = __fadd_rn(rays_o[ray * 3 + c], __fmul_rn(d[c], zz));   // render.py:49
          if (sl == 0) { e[0] = pt[0]; e[1] = pt[1]; e[2] = pt[2]; }
          else posenc_one_freq(pt, sl - 1, e + 3 + 6 * (sl - 1));
        } else {
          const float nrm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fmul_rn(d[2], d[2])));
          const float vd[3] = {__fdiv_rn(d[0], nrm), __fdiv_rn(d[1], nrm), __fdiv_rn(d[2], nrm)};    // render.py:37
          const int k = sl - (L_POS + 1);
          float* ed = e + CH_POS;
          if (k == 0) { ed[0] = vd[0]; ed[1] = vd[1]; ed[2] = vd[2]; }
          else posenc_one_freq(vd, k - 1, ed + 3 + 6 * (k - 1));
        }
      }
    }
    __syncthreads();
    const bool save = acts != nullptr;
    ActPlanes ap;
    if (save) {
      ap = act_planes(acts, m);
      for (int idx = tid; idx < rows_valid * CH_IN; idx += NT)            // column-major [90][M] (common.cuh ActPlanes)
        ap.emb[(int64_t)(idx / rows_valid) * m + row0 + idx % rows_valid] = E[(idx % rows_valid) * LDE + idx / rows_valid];
    }
#define ACT(plane, width) (save ? (plane) + row0 * (width) : nullptr), rows_valid

    // ---- trunk (dm_nerf.py:83-87)
    layer<true>(E, LDE, CH_POS, p.w[0], p.b[0], W_HID, X, LDX, Wt, ACT(ap.h[0], W_HID));
    for (int l = 1; l <= 4; ++l) layer<true>(X, LDX, W_HID, p.w[l], p.b[l], W_HID, X, LDX, Wt, ACT(ap.h[l], W_HID));
    for (int idx = tid; idx < TM * CH_POS; idx += NT) {           // skip: h = cat([h, pts])
      const int r = idx / CH_POS, c = idx % CH_POS;
      X[r * LDX + W_HID + c] = E[r * LDE + c];
    }
    __syncthreads();
    layer<true>(X, LDX, W_HID + CH_POS, p.w[5], p.b[5], W_HID, X, LDX, Wt, ACT(ap.h[5], W_HID));
    layer<true>(X, LDX, W_HID, p.w[6], p.b[6], W_HID, X, LDX, Wt, ACT(ap.h[6], W_HID));
    layer<true>(X, LDX, W_HID, p.w[7], p.b[7], W_HID, X, LDX, Wt, ACT(ap.h[7], W_HID));

    float* orow = out + row0 * C;
    // ---- density (dm_nerf.py:101) -> channel 3
    head(X, LDX, W_HID, p.w[L_DENSITY], p.b[L_DENSITY], 1, orow, C, 3, rows_valid);
    // ---- instance branch (dm_nerf.py:95-99,103) -> channels 4..
    layer<false>(X, LDX, W_HID, p.w[L_INS_FEAT], p.b[L_INS_FEAT], W_HID, B, LDB, Wt);
    // ---- colour branch (dm_nerf.py:89-93,102) -> channels 0..2   (h is dead after this layer: in place)
    layer<false>(X, LDX, W_HID, p.w[L_RGB_FEAT], p.b[L_RGB_FEAT], W_HID, X, LDX, Wt);
    for (int idx = tid; idx < TM * CH_DIR; idx += NT) {            // cat([rgb_feature, input_dirs])
      const int r = idx / CH_DIR, c = idx % CH_DIR;
      X[r * LDX + W_HID + c] = E[r * LDE + CH_POS + c];
    }
    __syncthreads();
    layer<true>(X, LDX, W_HID + CH_DIR, p.w[L_RGB_HID], p.b[L_RGB_HID], W_HID / 2, X, LDX, Wt, ACT(ap.rgb_hid, W_HID / 2));
    head(X, LDX, W_HID / 2, p.w[L_RGB_OUT], p.b[L_RGB_OUT], 3, orow, C, 0, rows_valid);
    layer<true>(B, LDB, W_HID, p.w[L_INS_HID], p.b[L_INS_HID], W_HID / 2, B, LDB, Wt, ACT(ap.ins_hid, W_HID / 2));
#undef ACT
    head(B, LDB, W_HID / 2, p.w[L_INS_OUT], p.b[L_INS_OUT], p.ins_num + 1, orow, C, 4, rows_valid);
  }
}
}  // namespace simt

int launch_mlp_simt(const NetParams& p, const float* x, const float* rays_o, const float* rays_d, const float* z,
                    int64_t m, int s, float* out, float* acts, cudaStream_t st) {
  DMN_CHECK((x != nullptr) != (rays_o != nullptr && rays_d != nullptr && z != nullptr),
            "mlp: pass either x or (rays_o, rays_d, z)");
  if (m == 0) return 0;
  static PerDeviceOnce attr_once;
  if (attr_once.first()) {
    DMN_CUDA(cudaFuncSetAttribute(simt::mlp_simt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)simt::SMEM_BYTES));
  }
  int dev = 0, sms = 0;
  DMN_CUDA(cudaGetDevice(&dev));
  DMN_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int64_t tiles = (m + simt::TM - 1) / simt::TM;
  const unsigned grid = (unsigned)(tiles < sms ? tiles : sms);
  simt::mlp_simt_kernel<<<grid, simt::NT, simt::SMEM_BYTES, st>>>(p, x, rays_o, rays_d, z, m, s, out, acts);
  DMN_LAUNCH_OK();
  return 0;
}

}  // namespace dmnerf
