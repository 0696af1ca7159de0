// Stand-alone per-ray stage kernels (one warp per ray): positional encoding, sigma->alpha warp-scan
// composite, inverse-CDF sampling, depth merge.  These back the piecewise C-ABI entry points
// (dmnerf_posenc / dmnerf_composite / dmnerf_sample_pdf / dmnerf_sort_concat) used by callers such as
// the reference's manipulator.py and mesh_generator.py, and the unfused render path.
#include "ray_ops.cuh"

namespace dmnerf {

constexpr int WARPS_PER_BLOCK = 4;

// ---------------------------------------------------------------- Embedder.embed (dm_nerf.py:37-38)
__global__ void posenc_kernel(const float* __restrict__ x, int64_t m, int L, float* __restrict__ out) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;     // one thread per (row, slot)
  const int slots = L + 1;
  if (idx >= m * slots) return;
  const int64_t row = idx / slots;
  const int k = (int)(idx % slots);
  const int od = 3 + 6 * L;
  const float v[3] = {x[row * 3 + 0], x[row * 3 + 1], x[row * 3 + 2]};
  float* o = out + row * od;
  if (k == 0) {
    o[0] = v[0]; o[1] = v[1]; o[2] = v[2];
  } else {
    float t[6];
    posenc_one_freq(v, k - 1, t);
#pragma unroll
    for (int c = 0; c < 6; ++c) o[3 + 6 * (k - 1) + c] = t[c];
  }
}

int launch_posenc(const float* x, int64_t m, int n_freqs, float* out, cudaStream_t st) {
  DMN_CHECK(n_freqs >= 0 && n_freqs <= 16, "posenc: n_freqs=%d out of range [0,16]", n_freqs);
  if (m == 0) return 0;
  const int64_t total = m * (n_freqs + 1);
  const int threads = 256;
  posenc_kernel<<<(unsigned)((total + threads - 1) / threads), threads, 0, st>>>(x, m, n_freqs, out);
  DMN_LAUNCH_OK();
  return 0;
}

// ---------------------------------------------------------------- render_train (render.py:6-28)
// One warp per ray.  Phase 1: warp-scan weights into shared memory.  Phase 2: one lane per output
// channel walks the samples in order (coalesced across channels), mirroring torch.sum(..., -2).
// SELECT: object selection -- a sample whose argmax_sigmoid label is not kept enters with density 0 (alpha = 0); raw is read,
// never edited.  With region.bits set (SELECT only) a sample the region drops (region_drops at o + d z) enters with alpha = 0
// too: the same test as the fused render kernels.  With an appearance table (SELECT only) a kept sample's density is scaled and
// its colour mapped by appearance_apply; the rgb lanes take the sample's label again from its logits.
template <bool SELECT>
__global__ void composite_kernel(const float* __restrict__ raw, const float* __restrict__ z,
                                 const float* __restrict__ rays_d, int64_t n, int S, int C, int keep_all,
                                 float* __restrict__ rgb, float* __restrict__ weights, float* __restrict__ depth,
                                 float* __restrict__ ins, float* __restrict__ acc, const ObjMask keep,
                                 const float* __restrict__ rays_o, const __grid_constant__ Region region,
                                 const float* __restrict__ appearance) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t ray = (int64_t)blockIdx.x * WARPS_PER_BLOCK + warp;
  if (ray >= n) return;
  float* w = smem + (size_t)warp * S;
  const float* zr = z + ray * S;
  const float* rr = raw + ray * S * C;
  const float dx = rays_d[ray * 3], dy = rays_d[ray * 3 + 1], dz = rays_d[ray * 3 + 2];
  const float dnorm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
  ray_weights(S, dnorm, [&](int i) {
    const float* ri = rr + (size_t)i * C;
    if constexpr (SELECT) {
      const int label = argmax_sigmoid(ri + 4, C - 4);
      if (!obj_kept(keep, label)) return 0.0f;
      if (region.bits) {
        const float o[3] = {rays_o[ray * 3], rays_o[ray * 3 + 1], rays_o[ray * 3 + 2]}, d[3] = {dx, dy, dz};
        float p[3];
        ray_point(o, d, zr[i], p);
        if (region_drops(region, label, p[0], p[1], p[2])) return 0.0f;
      }
      if (appearance) {
        float sg = fmaxf(ri[3], 0.0f), c[3] = {0.0f, 0.0f, 0.0f};
        appearance_apply(appearance, label, sg, c);
        return sg;                                 // >= 0: ray_weights' max(sigma, 0) leaves it as it is
      }
    }
    return ri[3];
  }, [&](int i) { return zr[i]; }, w, lane);
  __syncwarp();
  if (weights)
    for (int i = lane; i < S; i += 32) weights[ray * S + i] = w[i];
  const int n_ins_out = keep_all ? C - 4 : C - 5;
  for (int k = lane; k < C; k += 32) {
    if (k < 3) {
      float a = 0.0f;
      for (int i = 0; i < S; ++i) {
        float c = sigmoidf_acc(rr[(size_t)i * C + k]);
        if constexpr (SELECT) {
          if (appearance) {
            const float* ri = rr + (size_t)i * C;
            float sg = 0.0f, col[3] = {sigmoidf_acc(ri[0]), sigmoidf_acc(ri[1]), sigmoidf_acc(ri[2])};
            appearance_apply(appearance, argmax_sigmoid(ri + 4, C - 4), sg, col);
            c = k == 0 ? col[0] : (k == 1 ? col[1] : col[2]);
          }
        }
        a = __fadd_rn(a, __fmul_rn(w[i], c));
      }
      if (rgb) rgb[ray * 3 + k] = a;
    } else if (k == 3) {
      float d = 0.0f, s = 0.0f;
      for (int i = 0; i < S; ++i) {
        d = __fadd_rn(d, __fmul_rn(w[i], zr[i]));
        s = __fadd_rn(s, w[i]);
      }
      if (depth) depth[ray] = d;
      if (acc) acc[ray] = s;
    } else {
      float a = 0.0f;
      for (int i = 0; i < S; ++i) a = __fadd_rn(a, __fmul_rn(w[i], rr[(size_t)i * C + k]));
      if (ins && (k - 4) < n_ins_out) ins[ray * n_ins_out + (k - 4)] = sigmoidf_acc(a);
    }
  }
}

int launch_composite(const float* raw, const float* z, const float* rays_d, int64_t n, int s, int c, int keep_all,
                     float* rgb, float* weights, float* depth, float* ins, float* acc, cudaStream_t st, const Edit* edit,
                     const float* rays_o) {
  DMN_CHECK(s >= 1 && s <= 4096, "composite: n_samples=%d out of range [1,4096]", s);
  DMN_CHECK(c >= 5 && c <= 4 + DMNERF_MAX_INS + 1, "composite: channels=%d out of range", c);
  DMN_CHECK(!edit || !edit->region.bits || rays_o, "composite: a region needs the ray origins");
  if (n == 0) return 0;
  const size_t smem = (size_t)WARPS_PER_BLOCK * s * sizeof(float);
  auto kernel = edit ? composite_kernel<true> : composite_kernel<false>;
  if (smem > 48 * 1024)
    DMN_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const Edit none = {};
  const Edit& e = edit ? *edit : none;
  kernel<<<(unsigned)((n + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK), WARPS_PER_BLOCK * 32, smem, st>>>(
      raw, z, rays_d, n, s, c, keep_all, rgb, weights, depth, ins, acc, e.keep, rays_o, e.region, e.appearance);
  DMN_LAUNCH_OK();
  return 0;
}

// ---------------------------------------------------------------- sample_pdf (helpers.py:123-155)
__global__ void sample_pdf_kernel(const float* __restrict__ bins, const float* __restrict__ wts, int64_t n, int nb,
                                  int ns, const float* __restrict__ u, float* __restrict__ out) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t ray = (int64_t)blockIdx.x * WARPS_PER_BLOCK + warp;
  if (ray >= n) return;
  float* sb = smem + (size_t)warp * 2 * nb;
  float* cdf = sb + nb;
  for (int j = lane; j < nb; j += 32) sb[j] = bins[ray * nb + j];
  __syncwarp();
  const float* wr = wts + ray * (nb - 1);
  ray_sample_pdf(sb, [&](int j) { return wr[j]; }, nb, ns, u ? u + ray * ns : nullptr, cdf, out + ray * ns, lane);
}

int launch_sample_pdf(const float* bins, const float* weights, int64_t n, int nb, int ns, const float* u, float* out,
                      cudaStream_t st) {
  DMN_CHECK(nb >= 2 && nb <= 2048, "sample_pdf: n_bins=%d out of range [2,2048]", nb);
  DMN_CHECK(ns >= 2 && ns <= 4096, "sample_pdf: n_samples=%d out of range [2,4096]", ns);
  if (n == 0) return 0;
  const size_t smem = (size_t)WARPS_PER_BLOCK * 2 * nb * sizeof(float);
  if (smem > 48 * 1024)
    DMN_CUDA(cudaFuncSetAttribute(sample_pdf_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  sample_pdf_kernel<<<(unsigned)((n + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK), WARPS_PER_BLOCK * 32, smem, st>>>(
      bins, weights, n, nb, ns, u, out);
  DMN_LAUNCH_OK();
  return 0;
}

// ---------------------------------------------------------------- sort(cat(a, b)) (render.py:70)
__global__ void sort_concat_kernel(const float* __restrict__ a, const float* __restrict__ b, int64_t n, int na,
                                   int nb, float* __restrict__ out) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t ray = (int64_t)blockIdx.x * WARPS_PER_BLOCK + warp;
  if (ray >= n) return;
  const int T = na + nb;
  float* v = smem + (size_t)warp * T;
  for (int j = lane; j < na; j += 32) v[j] = a[ray * na + j];
  for (int j = lane; j < nb; j += 32) v[na + j] = b[ray * nb + j];
  __syncwarp();
  ray_rank_sort(v, T, out + ray * T, lane);
}

int launch_sort_concat(const float* a, const float* b, int64_t n, int na, int nb, float* out, cudaStream_t st) {
  DMN_CHECK(na >= 0 && nb >= 0 && na + nb >= 1 && na + nb <= 8192, "sort_concat: sizes %d+%d out of range", na, nb);
  if (n == 0) return 0;
  const size_t smem = (size_t)WARPS_PER_BLOCK * (na + nb) * sizeof(float);
  if (smem > 48 * 1024)
    DMN_CUDA(cudaFuncSetAttribute(sort_concat_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  sort_concat_kernel<<<(unsigned)((n + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK), WARPS_PER_BLOCK * 32, smem, st>>>(
      a, b, n, na, nb, out);
  DMN_LAUNCH_OK();
  return 0;
}

// ---------------------------------------------------------------- coarse depths (render.py:40-47)
// z_out[n, i] = z_in[i] (shared row or per-ray), jittered inside its stratum when t_rand is given.
__global__ void prep_z_kernel(const float* __restrict__ z_in, int64_t z_stride, const float* __restrict__ t_rand,
                              int64_t n, int S, float* __restrict__ z_out) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * S) return;
  const int64_t ray = idx / S;
  const int i = (int)(idx % S);
  const float* zr = z_in + ray * z_stride;
  float zi = zr[i];
  if (t_rand) {
    const float lower = (i == 0) ? zi : __fmul_rn(0.5f, __fadd_rn(zi, zr[i - 1]));
    const float upper = (i == S - 1) ? zi : __fmul_rn(0.5f, __fadd_rn(zr[i + 1], zi));
    zi = __fadd_rn(lower, __fmul_rn(__fsub_rn(upper, lower), t_rand[idx]));
  }
  z_out[idx] = zi;
}

int launch_prep_z(const float* z_in, int64_t z_stride, const float* t_rand, int64_t n, int s, float* z_out,
                  cudaStream_t st) {
  if (n == 0) return 0;
  const int64_t total = n * s;
  prep_z_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(z_in, z_stride, t_rand, n, s, z_out);
  DMN_LAUNCH_OK();
  return 0;
}

// ---------------------------------------------------------------- render.py:66-70 in one kernel
// z_mid, sample_pdf on weights[1:-1], concat with the coarse depths, sort.
__global__ void hier_sample_kernel(const float* __restrict__ z_c, const float* __restrict__ w_c,
                                   const float* __restrict__ u, int64_t n, int S, int NI, float* __restrict__ z_fine) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t ray = (int64_t)blockIdx.x * WARPS_PER_BLOCK + warp;
  if (ray >= n) return;
  const int nb = S - 1, T = S + NI;
  float* bins = smem + (size_t)warp * (2 * nb + T);
  float* cdf = bins + nb;
  float* vals = cdf + nb;                       // [S coarse | NI samples]
  const float* zr = z_c + ray * S;
  const float* wr = w_c + ray * S;
  for (int j = lane; j < S; j += 32) vals[j] = zr[j];
  __syncwarp();
  for (int j = lane; j < nb; j += 32) bins[j] = __fmul_rn(0.5f, __fadd_rn(vals[j + 1], vals[j]));   // render.py:66
  __syncwarp();
  ray_sample_pdf(bins, [&](int j) { return wr[j + 1]; }, nb, NI, u ? u + ray * NI : nullptr, cdf, vals + S, lane);
  // deterministic u gives two ascending runs (merge by binary search); random u -- or a last-bit inversion at a bin
  // boundary -- takes the general rank sort
  if (!u && ray_is_sorted(vals + S, NI, lane) && ray_is_sorted(vals, S, lane)) ray_merge_sorted(vals, S, vals + S, NI, z_fine + ray * T, lane);
  else ray_rank_sort(vals, T, z_fine + ray * T, lane);
}

int launch_hier_sample(const float* z_c, const float* w_c, const float* u, int64_t n, int s, int ni, float* z_fine,
                       cudaStream_t st) {
  DMN_CHECK(s >= 3 && s <= 1024 && ni >= 2 && ni <= 2048, "hier_sample: S=%d I=%d out of range", s, ni);
  if (n == 0) return 0;
  const size_t smem = (size_t)WARPS_PER_BLOCK * (2 * (s - 1) + s + ni) * sizeof(float);
  if (smem > 48 * 1024)
    DMN_CUDA(cudaFuncSetAttribute(hier_sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  hier_sample_kernel<<<(unsigned)((n + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK), WARPS_PER_BLOCK * 32, smem, st>>>(
      z_c, w_c, u, n, s, ni, z_fine);
  DMN_LAUNCH_OK();
  return 0;
}

// ---------------------------------------------------------------- get_rays_k (helpers.py:50-61)
struct Camera { float K[9]; float c2w[12]; };   // row-major 3x3 intrinsics, top 3x4 of the camera-to-world pose

__global__ void rays_kernel(Camera cam, int H, int W, float* __restrict__ rays_o, float* __restrict__ rays_d) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)H * W) return;
  const float i = (float)(idx % W), j = (float)(idx / W);                      // pixel column / row (exact linspace values)
  const float dx = __fdiv_rn(__fsub_rn(i, cam.K[2]), cam.K[0]);
  const float dy = __fdiv_rn(__fsub_rn(j, cam.K[5]), cam.K[4]);
  const float dz = cam.K[8];                                                    // K[2,2] * 1
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const float* R = cam.c2w + 4 * r;
    rays_d[idx * 3 + r] = __fadd_rn(__fadd_rn(__fmul_rn(dx, R[0]), __fmul_rn(dy, R[1])), __fmul_rn(dz, R[2]));
    rays_o[idx * 3 + r] = R[3];
  }
}

// Rays of selected pixels only (training: get_select_full / get_select_crop, helpers.py:64-111, keep 1024-3072 of the H*W
// rays of a frame): pix[i] = row * W + column of sample i.  Same arithmetic as rays_kernel, so the rows are bit-identical to
// get_rays_k(...)[row, column].
// c2w_dev != NULL: the pose is read from device memory (rows of 4 floats, c2w_ld apart) -- the training loop hands over a CUDA
// tensor (train_dmsr.py:27) and copying it to the host would synchronise every iteration.
__global__ void rays_at_kernel(Camera cam, const float* __restrict__ c2w_dev, int64_t c2w_ld, int W, const int64_t* __restrict__ pix,
                               int64_t n, float* __restrict__ rays_o, float* __restrict__ rays_d) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  if (c2w_dev) {
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) cam.c2w[4 * r + c] = __ldg(c2w_dev + r * c2w_ld + c);
  }
  const int64_t idx = pix[t];
  const float i = (float)(idx % W), j = (float)(idx / W);
  const float dx = __fdiv_rn(__fsub_rn(i, cam.K[2]), cam.K[0]);
  const float dy = __fdiv_rn(__fsub_rn(j, cam.K[5]), cam.K[4]);
  const float dz = cam.K[8];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const float* R = cam.c2w + 4 * r;
    rays_d[t * 3 + r] = __fadd_rn(__fadd_rn(__fmul_rn(dx, R[0]), __fmul_rn(dy, R[1])), __fmul_rn(dz, R[2]));
    rays_o[t * 3 + r] = R[3];
  }
}

int launch_rays_at(const float* K9, const float* c2w12, const float* c2w_dev, int64_t c2w_ld, int H, int W, const int64_t* pix,
                   int64_t n, float* rays_o, float* rays_d, cudaStream_t st) {
  DMN_CHECK(H >= 1 && W >= 1 && (int64_t)H * W <= (1LL << 31), "get_rays_at: bad image size %dx%d", H, W);
  if (n == 0) return 0;
  Camera cam;
  for (int i = 0; i < 9; ++i) cam.K[i] = K9[i];
  for (int i = 0; i < 12; ++i) cam.c2w[i] = c2w12 ? c2w12[i] : 0.0f;
  rays_at_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(cam, c2w_dev, c2w_ld, W, pix, n, rays_o, rays_d);
  DMN_LAUNCH_OK();
  return 0;
}

// n DISTINCT pseudo-random pixels of an H x W image without any host work: pix[i] = P(i), P a keyed bijection of [0, H*W)
// (6-round Feistel network on the next even power of two, cycle-walked back into range: at most 4 expected steps).  The
// uniform-without-replacement draw of helpers.py:100 (np.random.choice(H*W, N, replace=False)) costs the host a 307 200-element
// shuffle per iteration; this is the opt-in replacement (DMNERF_SELECT=device: NOT the reference's random stream).
__device__ __forceinline__ uint32_t mix32(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
  return x;
}
__global__ void select_pixels_kernel(uint64_t seed, uint32_t total, int half_bits, int64_t n, int64_t* __restrict__ pix) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const uint32_t mask = (1u << half_bits) - 1u;
  uint32_t x = (uint32_t)t;
  do {
    uint32_t l = x >> half_bits, r = x & mask;
#pragma unroll
    for (int round = 0; round < 6; ++round) {
      const uint32_t k = (uint32_t)(seed >> (8 * (round & 3))) ^ (uint32_t)(seed >> 32) * (2u * round + 1u);
      const uint32_t f = mix32(r ^ k ^ (0x9e3779b9u * (round + 1))) & mask;
      const uint32_t nl = r;
      r = l ^ f;
      l = nl;
    }
    x = (l << half_bits) | r;
  } while (x >= total);
  pix[t] = (int64_t)x;
}

int launch_select_pixels(uint64_t seed, int H, int W, int64_t n, int64_t* pix, cudaStream_t st) {
  const int64_t total = (int64_t)H * W;
  DMN_CHECK(H >= 1 && W >= 1 && total <= (1LL << 30), "select_pixels: bad image size %dx%d", H, W);
  DMN_CHECK(n >= 0 && n <= total, "select_pixels: %lld distinct pixels of %lld", (long long)n, (long long)total);
  if (n == 0) return 0;
  int bits = 1;
  while ((1LL << bits) < total) ++bits;
  const int half_bits = (bits + 1) / 2;
  select_pixels_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(seed, (uint32_t)total, half_bits, n, pix);
  DMN_LAUNCH_OK();
  return 0;
}

int launch_rays(const float* K9, const float* c2w12, int H, int W, float* rays_o, float* rays_d, cudaStream_t st) {
  DMN_CHECK(H >= 1 && W >= 1 && (int64_t)H * W <= (1LL << 31), "get_rays: bad image size %dx%d", H, W);
  Camera cam;
  for (int i = 0; i < 9; ++i) cam.K[i] = K9[i];
  for (int i = 0; i < 12; ++i) cam.c2w[i] = c2w12[i];
  const int64_t total = (int64_t)H * W;
  rays_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(cam, H, W, rays_o, rays_d);
  DMN_LAUNCH_OK();
  return 0;
}

}  // namespace dmnerf
