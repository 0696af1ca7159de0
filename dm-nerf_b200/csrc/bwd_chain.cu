// Gradient chain of the training backward (BASELINE config 4; reference train_dmsr.py:62-64, the dX half of
// total_loss.backward() through DM_NeRF.forward, networks/dm_nerf.py:80-106), with the heads folded like in the forward:
//     S1 | S2 = mask(rgb_hid) . (d_rgb W_rgb_out) | mask(ins_hid) . (d_ins W_ins_out)     (bwd_heads_kernel)
//     dY7 = mask(h7) . (S1 W_fold + d_sigma (x) w_density)      W_fold = W_rgb_hid[:, :256] W_rgb_feat  (folded heads)
//     dY(l-1) = mask(h(l-1)) . (dY(l) W(l)),  l = 7 .. 1        (the instance branch sees h.detach(): no trunk term)
// Every dX product is one split-bf16 wgmma GEMM (gemm_umma.cu) whose epilogue applies the ReLU mask from the 1-bit planes the
// training forward writes (ActPlanes::bits).  Each dY(l) is written once to HBM: those planes are what the per-layer dW GEMMs
// consume (a weight gradient needs all samples of one layer at once).
#include <cstring>

#include "common.cuh"
#include "umma_api.cuh"

namespace dmnerf {
namespace bk {

// ------------------------------------------------------------------------------------------------ head gradients
// d rgb_hid = mask . (d_rgb W_rgb_out), d ins_hid = mask . (d_ins W_ins_out)   (dm_nerf.py:102-103 backwards, K = 3 / ins_num+1)
// written side by side into one [M,256] plane so that ONE dW GEMM against h7 serves both branches.
// A warp handles 8 rows, a lane 4 adjacent hidden units of both halves (float4 weights from shared memory, float4 broadcasts of the
// staged d_out rows, 512 contiguous bytes per warp store).  The rows of d_out are staged zero-padded to a multiple of 4
// channels.  (The first version -- one thread per unit, one scalar shared-memory load per multiply-add -- was bound by the
// shared-memory load unit, not by the 268 MB it writes.)
constexpr int HEAD_ROWS = 8;        // rows per warp and iteration
constexpr int HEAD_BLOCK_ROWS = 4 * HEAD_ROWS;
__global__ void __launch_bounds__(128) bwd_heads_kernel(const float* __restrict__ d_out, int C, int64_t m, const float* __restrict__ w_rgb,
                                                        const float* __restrict__ w_ins, int ins1, const uint16_t* __restrict__ bits,
                                                        float* __restrict__ s12, int rows_per_block) {
  extern __shared__ __align__(16) float sm[];
  const int ins4 = (ins1 + 3) & ~3;       // instance channels padded to a multiple of 4 (zero weights)
  const int CP = 4 + ins4;                // staged row: rgb, sigma, padded instance channels
  float* wi = sm;                         // [ins4][128]
  float* drow = wi + ins4 * 128;          // [HEAD_BLOCK_ROWS][CP]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int k = 0; k < ins4; ++k) wi[k * 128 + tid] = (k < ins1) ? w_ins[k * 128 + tid] : 0.0f;
  const float* wl = w_rgb + 4 * lane;     // scalar loads: a parameter tensor need not be 16-byte aligned
  const float4 wr0 = make_float4(wl[0], wl[1], wl[2], wl[3]), wr1 = make_float4(wl[128], wl[129], wl[130], wl[131]),
               wr2 = make_float4(wl[256], wl[257], wl[258], wl[259]);
  const float4* wi4 = reinterpret_cast<const float4*>(wi) + lane;       // + k * 32: units 4 lane .. 4 lane + 3 of channel k
  const int64_t r0 = (int64_t)blockIdx.x * rows_per_block;
  const int64_t r1 = (r0 + rows_per_block < m) ? r0 + rows_per_block : m;
  for (int64_t row = r0; row < r1; row += HEAD_BLOCK_ROWS) {
    const int nr = (int)((r1 - row < HEAD_BLOCK_ROWS) ? r1 - row : HEAD_BLOCK_ROWS);
    __syncthreads();
    for (int i = tid; i < HEAD_BLOCK_ROWS * CP; i += 128) {
      const int q = i / CP, c = i - q * CP;
      drow[i] = (q < nr && c < C) ? d_out[(row + q) * C + c] : 0.0f;
    }
    __syncthreads();
    const float4* d4 = reinterpret_cast<const float4*>(drow) + warp * HEAD_ROWS * (CP / 4);
    float4 a1[HEAD_ROWS], a2[HEAD_ROWS];
#pragma unroll
    for (int q = 0; q < HEAD_ROWS; ++q) {
      const float4 d = d4[q * (CP / 4)];
      // per unit the same order as a scalar loop over the channels: ((0 + x w0) + y w1) + z w2
      a1[q].x = fmaf(d.z, wr2.x, fmaf(d.y, wr1.x, __fmul_rn(d.x, wr0.x)));
      a1[q].y = fmaf(d.z, wr2.y, fmaf(d.y, wr1.y, __fmul_rn(d.x, wr0.y)));
      a1[q].z = fmaf(d.z, wr2.z, fmaf(d.y, wr1.z, __fmul_rn(d.x, wr0.z)));
      a1[q].w = fmaf(d.z, wr2.w, fmaf(d.y, wr1.w, __fmul_rn(d.x, wr0.w)));
      a2[q] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    }
    for (int k4 = 0; k4 < ins4 / 4; ++k4) {
      const float4 w0 = wi4[(4 * k4) * 32], w1 = wi4[(4 * k4 + 1) * 32], w2 = wi4[(4 * k4 + 2) * 32], w3 = wi4[(4 * k4 + 3) * 32];
#pragma unroll
      for (int q = 0; q < HEAD_ROWS; ++q) {
        const float4 d = d4[q * (CP / 4) + 1 + k4];
        a2[q].x = fmaf(d.w, w3.x, fmaf(d.z, w2.x, fmaf(d.y, w1.x, fmaf(d.x, w0.x, a2[q].x))));
        a2[q].y = fmaf(d.w, w3.y, fmaf(d.z, w2.y, fmaf(d.y, w1.y, fmaf(d.x, w0.y, a2[q].y))));
        a2[q].z = fmaf(d.w, w3.z, fmaf(d.z, w2.z, fmaf(d.y, w1.z, fmaf(d.x, w0.z, a2[q].z))));
        a2[q].w = fmaf(d.w, w3.w, fmaf(d.z, w2.w, fmaf(d.y, w1.w, fmaf(d.x, w0.w, a2[q].w))));
      }
    }
    const int sh = (lane & 3) * 4;          // this lane's 4 units inside their 16-unit mask group (lane >> 2)
#pragma unroll
    for (int q = 0; q < HEAD_ROWS; ++q) {
      const int lr = warp * HEAD_ROWS + q;
      if (lr >= nr) break;
      const int64_t rq = row + lr;
      const uint32_t br = (uint32_t)bits[act_bits_index(8, lane >> 2, rq, m)] >> sh, bi = (uint32_t)bits[act_bits_index(9, lane >> 2, rq, m)] >> sh;
      float4 o1 = a1[q], o2 = a2[q];
      if (!(br & 1u)) o1.x = 0.0f;
      if (!(br & 2u)) o1.y = 0.0f;
      if (!(br & 4u)) o1.z = 0.0f;
      if (!(br & 8u)) o1.w = 0.0f;
      if (!(bi & 1u)) o2.x = 0.0f;
      if (!(bi & 2u)) o2.y = 0.0f;
      if (!(bi & 4u)) o2.z = 0.0f;
      if (!(bi & 8u)) o2.w = 0.0f;
      *reinterpret_cast<float4*>(s12 + rq * 256 + 4 * lane) = o1;               // one [M,256] plane: d rgb_hid | d ins_hid
      *reinterpret_cast<float4*>(s12 + rq * 256 + 128 + 4 * lane) = o2;
    }
  }
}

// ReLU masks from saved fp32 activation planes (exact-fp32 CUDA-core forward: it does not write ActPlanes::bits itself).
__global__ void mask_bits_kernel(const float* __restrict__ plane, int width, int64_t m, uint16_t* __restrict__ bits, int pl) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;       // one thread per (group, row), rows fastest
  const int groups = width / 16;
  if (idx >= m * groups) return;
  const int g = (int)(idx / m);
  const int64_t row = idx % m;
  const float4* src = reinterpret_cast<const float4*>(plane + row * width + g * 16);
  uint32_t b = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 q = __ldg(src + i);
    b |= (q.x > 0.0f ? 1u : 0u) << (4 * i) | (q.y > 0.0f ? 1u : 0u) << (4 * i + 1) | (q.z > 0.0f ? 1u : 0u) << (4 * i + 2) |
         (q.w > 0.0f ? 1u : 0u) << (4 * i + 3);
  }
  bits[act_bits_index(pl, g, row, m)] = (uint16_t)b;
}

// dY7 before the mask: d sigma (x) density_linear.weight (dm_nerf.py:101 backwards); the folded rgb head is added by the GEMM.
__global__ void dsig_outer_kernel(const float* __restrict__ d_out, int C, const float* __restrict__ w_dens, int64_t m,
                                  float* __restrict__ dy7) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;      // one thread per 4 units of a row
  if (idx >= m * 64) return;
  const int64_t row = idx >> 6;
  const int u = (int)(idx & 63) * 4;
  const float d = __ldg(d_out + row * C + 3);
  *reinterpret_cast<float4*>(dy7 + row * 256 + u) =
      make_float4(d * __ldg(w_dens + u), d * __ldg(w_dens + u + 1), d * __ldg(w_dens + u + 2), d * __ldg(w_dens + u + 3));
}

}  // namespace bk

// ================================================================================================ host
int launch_mask_bits(float* acts, int64_t m, cudaStream_t st) {
  const ActPlanes ap = act_planes(acts, m);
  for (int pl = 0; pl < 10; ++pl) {
    const float* src = pl < 8 ? ap.h[pl] : (pl == 8 ? ap.rgb_hid : ap.ins_hid);
    const int width = pl < 8 ? W_HID : W_HID / 2;
    const int64_t total = m * (width / 16);
    bk::mask_bits_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(src, width, m, ap.bits, pl);
    DMN_LAUNCH_OK();
  }
  return 0;
}

int launch_bwd_heads(const NetParams& p, const float* d_out, int64_t m, const uint16_t* bits, float* s12, cudaStream_t st) {
  const int ins1 = p.ins_num + 1, C = 4 + ins1;
  if (m == 0) return 0;
  const int rows = 64;
  const int ins4 = (ins1 + 3) & ~3;
  const size_t smem = (size_t)(ins4 * 128 + bk::HEAD_BLOCK_ROWS * (4 + ins4)) * sizeof(float);
  static PerDeviceOnce once;
  if (once.first()) DMN_CUDA(cudaFuncSetAttribute(bk::bwd_heads_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
  bk::bwd_heads_kernel<<<(unsigned)((m + rows - 1) / rows), 128, smem, st>>>(d_out, C, m, p.w[L_RGB_OUT], p.w[L_INS_OUT], ins1, bits, s12,
                                                                           rows);
  DMN_LAUNCH_OK();
  return 0;
}

// dY(7..0) of one network from d rgb_hid (s1, row stride 256) and d sigma (column 3 of d_out).  dy: 8 planes [m,256].
int launch_bwd_chain(const UmmaWeights& w, const NetParams& p, const float* s1, const float* d_out, const ActPlanes& ap, int64_t m,
                     float* const* dy, cudaStream_t st) {
  DMN_CHECK(w.ready && w.extra, "bwd_chain: weights not packed (call dmnerf_set_weights first)");
  if (m == 0) return 0;
  const int C = 4 + p.ins_num + 1;
  bk::dsig_outer_kernel<<<(unsigned)((m * 64 + 255) / 256), 256, 0, st>>>(d_out, C, p.w[L_DENSITY], m, dy[7]);
  DMN_LAUNCH_OK();
  auto bits = [&](int plane) { return ap.bits + (int64_t)plane * ACT_BITS_GROUPS * m; };
  int rc = launch_gemm_nn_tc(s1, 256, umma_fold_w_rgb(w), 283, dy[7], 256, m, 128, 1, nullptr, nullptr, 0, st, bits(7));
  for (int l = 7; l >= 1 && rc == 0; --l)
    rc = launch_gemm_nn_tc(dy[l], 256, p.w[l], layer_in(l), dy[l - 1], 256, m, 256, 0, nullptr, nullptr, 0, st, bits(l - 1));
  return rc;
}

}  // namespace dmnerf
