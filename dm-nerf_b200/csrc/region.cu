// Region builders (DESIGN.md, "Region selection"): the packed bit grid a render reads per sample, from a component id grid
// (pack), grown by binary dilation (dilate), and the per-point test of the render kernels on its own (contains).
// Bits: grid point v = (i dim + j) dim + k is bit v & 31 of word v >> 5; the bits past dim^3 of the last word are 0.
#include <cmath>

#include "ray_ops.cuh"

namespace dmnerf {

namespace {

constexpr int RG_THREADS = 256;

__device__ __forceinline__ int64_t stride_of() { return (int64_t)gridDim.x * blockDim.x; }

int blocks_for(int64_t n) {
  const int64_t b = (n + RG_THREADS - 1) / RG_THREADS;
  const int64_t cap = 1 << 20;
  return (int)(b < 1 ? 1 : (b < cap ? b : cap));
}

// pack: one warp per word (32 consecutive points), bit = the point's id is set in the table (ids outside [0, n_ids) give 0)
__global__ void __launch_bounds__(RG_THREADS) region_pack_kernel(const int32_t* __restrict__ ids, int64_t n,
                                                                 const uint32_t* __restrict__ table, int64_t n_ids,
                                                                 uint32_t* __restrict__ bits) {
  const int lane = threadIdx.x & 31;
  // the stride is a multiple of 32, so a warp always holds the aligned points 32 q .. 32 q + 31
  for (int64_t base = (int64_t)blockIdx.x * RG_THREADS + (threadIdx.x & ~31); base < n; base += stride_of()) {
    const int64_t p = base + lane;
    bool on = false;
    if (p < n) {
      const int id = ids[p];
      on = id >= 0 && id < n_ids && ((__ldg(table + (id >> 5)) >> (id & 31)) & 1u);
    }
    const uint32_t word = __ballot_sync(0xffffffffu, on);
    if (lane == 0) bits[base >> 5] = word;
  }
}

__device__ __forceinline__ bool bit_at(const uint32_t* bits, int64_t v) { return (__ldcg(bits + (v >> 5)) >> (v & 31)) & 1u; }

// one dilation step: a point is set when it or one of its neighbours (6: faces, 26: faces, edges and corners) is set; neighbours
// outside the grid count as 0 (never wrapped).  invert: the complement is written (last step only).
template <int CONN>
__global__ void __launch_bounds__(RG_THREADS) region_dilate_kernel(const uint32_t* __restrict__ in, int dim, int64_t n, int invert,
                                                                   uint32_t* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  for (int64_t base = (int64_t)blockIdx.x * RG_THREADS + (threadIdx.x & ~31); base < n; base += stride_of()) {
    const int64_t p = base + lane;
    bool on = false;
    if (p < n) {
      const int k = (int)(p % dim), j = (int)((p / dim) % dim), i = (int)(p / ((int64_t)dim * dim));
      on = bit_at(in, p);
      for (int di = -1; di <= 1 && !on; ++di) {
        const int ni = i + di;
        if (ni < 0 || ni >= dim) continue;
        for (int dj = -1; dj <= 1 && !on; ++dj) {
          const int nj = j + dj;
          if (nj < 0 || nj >= dim) continue;
          for (int dk = -1; dk <= 1 && !on; ++dk) {
            const int nk = k + dk;
            if (nk < 0 || nk >= dim) continue;
            if (CONN == 6 && (di != 0) + (dj != 0) + (dk != 0) != 1) continue;
            on = bit_at(in, ((int64_t)ni * dim + nj) * dim + nk);
          }
        }
      }
      if (invert) on = !on;
    }
    const uint32_t word = __ballot_sync(0xffffffffu, on);
    if (lane == 0) out[base >> 5] = word;
  }
}

// invert without dilation: the complement, the tail bits of the last word kept 0
__global__ void __launch_bounds__(RG_THREADS) region_invert_kernel(const uint32_t* __restrict__ in, int64_t n, uint32_t* __restrict__ out) {
  const int64_t words = (n + 31) / 32;
  for (int64_t w = (int64_t)blockIdx.x * RG_THREADS + threadIdx.x; w < words; w += stride_of()) {
    const int64_t used = n - 32 * w;
    const uint32_t mask = used >= 32 ? 0xffffffffu : ((1u << used) - 1u);
    out[w] = ~in[w] & mask;
  }
}

__global__ void __launch_bounds__(RG_THREADS) region_contains_kernel(const Region r, const float* __restrict__ pts, int64_t n,
                                                                     uint8_t* __restrict__ out) {
  for (int64_t q = (int64_t)blockIdx.x * RG_THREADS + threadIdx.x; q < n; q += stride_of())
    out[q] = region_bit(r, pts[3 * q], pts[3 * q + 1], pts[3 * q + 2]) == 1 ? 1 : 0;
}

}  // namespace

int region_check(int dim, const float* map12, const char* who) {
  DMN_CHECK(dim >= 2 && dim <= REGION_MAX_DIM, "%s: dim %d out of range [2, %d] (dim^3 must stay below 2^31)", who, dim,
            REGION_MAX_DIM);
  if (map12)
    for (int i = 0; i < 12; ++i) DMN_CHECK(std::isfinite(map12[i]), "%s: voxel map entry %d is not finite", who, i);
  return 0;
}

int region_from_abi(const dmnerf_region& d, Region& r, const char* who) {
  DMN_CHECK(d.bits != nullptr, "%s: a region with NULL bits", who);
  if (region_check(d.dim, d.voxel_map, who)) return 1;
  r = Region{};
  r.bits = d.bits;
  for (int i = 0; i < 12; ++i) r.map[i] = d.voxel_map[i];
  r.dim = d.dim;
  r.outside_keep = d.outside_keep ? 1 : 0;
  for (int i = 0; i < 4; ++i) r.applies.w[i] = d.applies[i];
  return 0;
}

int region_pack(const int32_t* ids, int dim, const uint32_t* table, int64_t n_ids, uint32_t* bits, cudaStream_t st) {
  const char* who = "region_pack";
  if (region_check(dim, nullptr, who)) return 1;
  DMN_CHECK(ids && bits, "%s: NULL ids / bits", who);
  DMN_CHECK(n_ids >= 0 && (n_ids == 0 || table), "%s: n_ids %lld needs a table", who, (long long)n_ids);
  const int64_t n = (int64_t)dim * dim * dim;
  region_pack_kernel<<<blocks_for(n), RG_THREADS, 0, st>>>(ids, n, table, n_ids, bits);
  DMN_LAUNCH_OK();
  return 0;
}

int region_dilate(const uint32_t* in, int dim, int r, int connectivity, int invert, uint32_t* out, uint32_t* tmp, cudaStream_t st) {
  const char* who = "region_dilate";
  if (region_check(dim, nullptr, who)) return 1;
  DMN_CHECK(in && out, "%s: NULL bits", who);
  DMN_CHECK(r >= 0, "%s: radius %d is negative", who, r);
  DMN_CHECK(connectivity == 6 || connectivity == 26, "%s: connectivity %d is not 6 or 26", who, connectivity);
  DMN_CHECK(in != out || r == 0, "%s: in and out must be distinct buffers", who);
  DMN_CHECK(r < 2 || (tmp && tmp != in && tmp != out), "%s: a radius of 2 or more needs a separate scratch buffer", who);
  const int64_t n = (int64_t)dim * dim * dim, words = region_words(dim);
  if (r == 0) {
    if (invert) {
      region_invert_kernel<<<blocks_for(words), RG_THREADS, 0, st>>>(in, n, out);
      DMN_LAUNCH_OK();
    } else if (in != out) {
      DMN_CUDA(cudaMemcpyAsync(out, in, (size_t)words * sizeof(uint32_t), cudaMemcpyDeviceToDevice, st));
    }
    return 0;
  }
  // steps alternate between out and tmp so that the last one lands in out
  const uint32_t* src = in;
  for (int s = 0; s < r; ++s) {
    uint32_t* dst = ((r - 1 - s) & 1) ? tmp : out;
    const int inv = (s == r - 1) ? invert : 0;
    if (connectivity == 6) region_dilate_kernel<6><<<blocks_for(n), RG_THREADS, 0, st>>>(src, dim, n, inv, dst);
    else region_dilate_kernel<26><<<blocks_for(n), RG_THREADS, 0, st>>>(src, dim, n, inv, dst);
    DMN_LAUNCH_OK();
    src = dst;
  }
  return 0;
}

int region_contains(const Region& r, const float* pts, int64_t n, uint8_t* out, cudaStream_t st) {
  DMN_CHECK(n >= 0 && (n == 0 || (pts && out)), "region_contains: bad points");
  if (n == 0) return 0;
  region_contains_kernel<<<blocks_for(n), RG_THREADS, 0, st>>>(r, pts, n, out);
  DMN_LAUNCH_OK();
  return 0;
}

}  // namespace dmnerf
