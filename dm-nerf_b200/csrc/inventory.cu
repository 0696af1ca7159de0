// Object inventory (DESIGN.md, "Object inventory"): per-group reductions over the solid points (occ > level) of a labelled
// occupancy grid.  Two passes over the grid [dim]^3 (C order, index (i, j, k)):
//   voxels: per group the solid count, the three per-axis index histograms and the 9 integer index moments;
//   spans:  per group the min / max of three fp64 projections s = u . (i, j, k) + o of the group's points.
// Every sum is an integer and every span a min / max of ordered 64-bit keys, so the results do not depend on the launch shape or
// on the order of the atomics: two calls give the same bits.  A block walks tiles of one i-plane, 32 rows (j) x 32 columns (k);
// each warp owns a row at a time, lane = column.  Shared-memory counters are aggregated over a warp where the warp's solid points
// share one label (the common case: neighbouring points belong to one object), and a tile's counters reach global memory once
// per touched label and counter.
#include <cmath>
#include <cstring>
#include <vector>

#include "common.cuh"

namespace dmnerf {

constexpr int TILE = 32;                      // tile edge along j and k (a warp spans the k edge)
constexpr int WARPS = 8;                      // a warp takes rows w, w + 8, w + 16, w + 24 of a tile
constexpr int THREADS = 32 * WARPS;
constexpr int N_MOM = 10;                     // count, Si, Sj, Sk, Sii, Sjj, Skk, Sij, Sik, Sjk
constexpr unsigned FULL = 0xffffffffu;

enum { INV_BAD_NAN = 1, INV_BAD_LABEL = 2 };

struct InvTiling {
  int dim, tiles_1d;
  int64_t n_tiles;
  __device__ void tile(int64_t t, int& i, int& j0, int& k0) const {
    const int64_t per_plane = (int64_t)tiles_1d * tiles_1d;
    i = (int)(t / per_plane);
    const int r = (int)(t % per_plane);
    j0 = (r / tiles_1d) * TILE;
    k0 = (r % tiles_1d) * TILE;
  }
};

// the grid point of lane / row (j, k): inside the grid?  If so its label (validated) and whether it is one of its group's points
struct InvPoint {
  bool solid;
  int label;
};

__device__ __forceinline__ InvPoint classify(const float* __restrict__ occ, const int16_t* __restrict__ labels, int64_t p, float level,
                                          int n_labels, const int* __restrict__ box, int i, int j, int k, int* bad) {
  const float v = occ[p];
  const int lab = labels ? (int)labels[p] : 0;
  if (v != v) atomicOr(bad, INV_BAD_NAN);
  if (lab < 0 || lab >= n_labels) {
    atomicOr(bad, INV_BAD_LABEL);
    return {false, 0};
  }
  bool in = v > level;
  if (in && box) {
    const int* b = box + 6 * lab;
    in = i >= b[0] && i <= b[1] && j >= b[2] && j <= b[3] && k >= b[4] && k <= b[5];
  }
  return {in, lab};
}

// the label every solid lane of the warp shares, or -1 when they differ (or none is solid)
__device__ __forceinline__ int warp_common_label(const InvPoint& pt) {
  const unsigned solid = __ballot_sync(FULL, pt.solid);
  if (!solid) return -1;
  const int first = __shfl_sync(FULL, pt.label, __ffs(solid) - 1);
  return __all_sync(FULL, !pt.solid || pt.label == first) ? first : -1;
}

// ---- voxels -------------------------------------------------------------------------------------------------------------
// shared, per label: jh [32] (row counts of the tile), kh [32] (column counts), sjk (sum of jl * kl, tile-local indices), touched
__global__ void __launch_bounds__(THREADS) object_voxels_kernel(const float* __restrict__ occ, const int16_t* __restrict__ labels,
                                                                 InvTiling tl, float level, int n_labels, const int* __restrict__ boxes,
                                                                 unsigned long long* __restrict__ mom, uint32_t* __restrict__ hist,
                                                                 int* bad) {
  extern __shared__ uint32_t sh[];
  uint32_t* jh = sh;                                   // [n_labels][32]
  uint32_t* kh = jh + n_labels * TILE;                 // [n_labels][32]
  uint32_t* sjk = kh + n_labels * TILE;                // [n_labels]
  uint32_t* touched = sjk + n_labels;                  // [n_labels]
  int* box = reinterpret_cast<int*>(touched + n_labels);   // [n_labels][6] when boxes
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int q = threadIdx.x; q < n_labels * (2 * TILE + 2); q += THREADS) sh[q] = 0;
  if (boxes)
    for (int q = threadIdx.x; q < 6 * n_labels; q += THREADS) box[q] = boxes[q];
  __syncthreads();
  const int dim = tl.dim;
  const int64_t d = dim;
  for (int64_t t = blockIdx.x; t < tl.n_tiles; t += gridDim.x) {
    int i, j0, k0;
    tl.tile(t, i, j0, k0);
    const int k = k0 + lane;
    for (int jl = warp; jl < TILE; jl += WARPS) {
      const int j = j0 + jl;
      if (j >= dim) break;                                                   // warp-uniform
      InvPoint pt{false, 0};
      if (k < dim) pt = classify(occ, labels, ((int64_t)i * d + j) * d + k, level, n_labels, boxes ? box : nullptr, i, j, k, bad);
      if (pt.solid) atomicAdd(kh + pt.label * TILE + lane, 1u);            // distinct columns within a warp
      const int common = warp_common_label(pt);
      if (common >= 0) {
        const unsigned solid = __ballot_sync(FULL, pt.solid);
        unsigned skl = pt.solid ? (unsigned)lane : 0u;
#pragma unroll
        for (int o = 16; o; o >>= 1) skl += __shfl_xor_sync(FULL, skl, o);
        if (lane == 0) {
          atomicAdd(jh + common * TILE + jl, (uint32_t)__popc(solid));
          atomicAdd(sjk + common, (uint32_t)jl * skl);
          touched[common] = 1;
        }
      } else if (pt.solid) {
        atomicAdd(jh + pt.label * TILE + jl, 1u);
        atomicAdd(sjk + pt.label, (uint32_t)(jl * lane));
        touched[pt.label] = 1;
      }
    }
    __syncthreads();
    // flush: warp w takes labels w, w + 8, ...; lane = tile-local row (jh) and column (kh) index
    for (int l = warp; l < n_labels; l += WARPS) {
      if (!touched[l]) continue;                                           // warp-uniform
      const uint32_t a = jh[l * TILE + lane], b = kh[l * TILE + lane];
      const uint32_t x = (uint32_t)lane;
      uint32_t c = a, sj = x * a, sjj = x * x * a, sk = x * b, skk = x * x * b;
#pragma unroll
      for (int o = 16; o; o >>= 1) {
        c += __shfl_xor_sync(FULL, c, o);
        sj += __shfl_xor_sync(FULL, sj, o);
        sjj += __shfl_xor_sync(FULL, sjj, o);
        sk += __shfl_xor_sync(FULL, sk, o);
        skk += __shfl_xor_sync(FULL, skk, o);
      }
      uint32_t* hl = hist + (int64_t)l * 3 * dim;
      if (a) atomicAdd(hl + dim + j0 + lane, a);
      if (b) atomicAdd(hl + 2 * dim + k0 + lane, b);
      if (lane == 0) {
        typedef unsigned long long u64;
        const u64 n = c, I = (u64)i, J = (u64)j0, K = (u64)k0;
        const u64 Sj = J * n + sj, Sk = K * n + sk;
        const u64 Sjj = J * J * n + 2 * J * sj + sjj, Skk = K * K * n + 2 * K * sk + skk;
        const u64 Sjk = J * K * n + J * sk + K * sj + sjk[l];
        const u64 v[N_MOM] = {n, I * n, Sj, Sk, I * I * n, Sjj, Skk, I * Sj, I * Sk, Sjk};
        u64* m = mom + (int64_t)l * N_MOM;
#pragma unroll
        for (int q = 0; q < N_MOM; ++q) atomicAdd(m + q, v[q]);
        atomicAdd(hl + i, c);
        sjk[l] = 0;
        touched[l] = 0;
      }
      jh[l * TILE + lane] = 0;
      kh[l * TILE + lane] = 0;
    }
    __syncthreads();
  }
}

// ---- spans ---------------------------------------------------------------------------------------------------------------
// a double as a signed 64-bit key of the same order (negative values: magnitude bits flipped)
__device__ __forceinline__ long long order_key(double x) {
  const long long b = __double_as_longlong(x);
  return b >= 0 ? b : b ^ 0x7fffffffffffffffLL;
}

// shared, per label: keys [3][2] (min, max of each projection) and touched; per label in constant-like global memory: u [3][4]
__global__ void __launch_bounds__(THREADS) object_spans_kernel(const float* __restrict__ occ, const int16_t* __restrict__ labels,
                                                                InvTiling tl, float level, int n_labels, const int* __restrict__ boxes,
                                                                const double* __restrict__ axes, long long* __restrict__ keys,
                                                                int* bad) {
  extern __shared__ long long shk[];
  long long* sk = shk;                                             // [n_labels][6]
  int* touched = reinterpret_cast<int*>(sk + 6 * n_labels);       // [n_labels]
  int* box = touched + n_labels;                                  // [n_labels][6]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long KMIN0 = 0x7ff0000000000000LL;                   // order_key(+inf): the empty minimum
  const long long KMAX0 = (long long)0x800fffffffffffffULL;       // order_key(-inf): the empty maximum
  for (int q = threadIdx.x; q < 6 * n_labels; q += THREADS) {
    sk[q] = (q & 1) ? KMAX0 : KMIN0;
    box[q] = boxes[q];
  }
  for (int q = threadIdx.x; q < n_labels; q += THREADS) touched[q] = 0;
  __syncthreads();
  const int dim = tl.dim;
  const int64_t d = dim;
  for (int64_t t = blockIdx.x; t < tl.n_tiles; t += gridDim.x) {
    int i, j0, k0;
    tl.tile(t, i, j0, k0);
    const int k = k0 + lane;
    for (int jl = warp; jl < TILE; jl += WARPS) {
      const int j = j0 + jl;
      if (j >= dim) break;
      InvPoint pt{false, 0};
      if (k < dim) pt = classify(occ, labels, ((int64_t)i * d + j) * d + k, level, n_labels, box, i, j, k, bad);
      const int common = warp_common_label(pt);
      long long kv[6];
      const int lab = pt.solid ? pt.label : (common >= 0 ? common : 0);
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        const double* u = axes + (lab * 3 + a) * 4;
        // ((u0 i + u1 j) + u2 k) + o, each operation rounded once (no contraction): the host twin repeats it exactly
        const double s = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(u[0], (double)i), __dmul_rn(u[1], (double)j)),
                                             __dmul_rn(u[2], (double)k)), u[3]);
        const long long key = order_key(s);
        kv[2 * a] = pt.solid ? key : KMIN0;
        kv[2 * a + 1] = pt.solid ? key : KMAX0;
      }
      if (common >= 0) {
#pragma unroll
        for (int o = 16; o; o >>= 1)
#pragma unroll
          for (int a = 0; a < 3; ++a) {
            const long long lo = __shfl_xor_sync(FULL, kv[2 * a], o), hi = __shfl_xor_sync(FULL, kv[2 * a + 1], o);
            kv[2 * a] = lo < kv[2 * a] ? lo : kv[2 * a];
            kv[2 * a + 1] = hi > kv[2 * a + 1] ? hi : kv[2 * a + 1];
          }
        if (lane == 0) {
          long long* s = sk + 6 * common;
#pragma unroll
          for (int a = 0; a < 3; ++a) {
            atomicMin(s + 2 * a, kv[2 * a]);
            atomicMax(s + 2 * a + 1, kv[2 * a + 1]);
          }
          touched[common] = 1;
        }
      } else if (pt.solid) {
        long long* s = sk + 6 * pt.label;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          atomicMin(s + 2 * a, kv[2 * a]);
          atomicMax(s + 2 * a + 1, kv[2 * a + 1]);
        }
        touched[pt.label] = 1;
      }
    }
  }
  __syncthreads();
  // once per block: the touched labels' keys
  for (int q = threadIdx.x; q < 6 * n_labels; q += THREADS) {
    if (!touched[q / 6]) continue;
    if (q & 1) atomicMax(keys + q, sk[q]);
    else atomicMin(keys + q, sk[q]);
  }
}

static double key_value(long long key) {
  const long long b = key >= 0 ? key : key ^ 0x7fffffffffffffffLL;
  double x;
  memcpy(&x, &b, sizeof(x));
  return x;
}

static int check_args(const float* occ, int dim, int n_labels, const char* who) {
  DMN_CHECK(occ != nullptr, "%s: occ is NULL", who);
  DMN_CHECK(dim >= 2 && dim <= 2048, "%s: dim %d out of range [2, 2048]", who, dim);
  DMN_CHECK(n_labels >= 1 && n_labels <= DMNERF_MAX_INS + 1, "%s: n_labels %d out of range [1, %d]", who, n_labels,
            DMNERF_MAX_INS + 1);
  return 0;
}

static InvTiling tiling(int dim) {
  InvTiling t;
  t.dim = dim;
  t.tiles_1d = (dim + TILE - 1) / TILE;
  t.n_tiles = (int64_t)dim * t.tiles_1d * t.tiles_1d;
  return t;
}

static int grid_blocks(const InvTiling& t, size_t smem, const void* kernel) {
  int dev = 0, sms = 0, per_sm = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, THREADS, smem) != cudaSuccess || per_sm < 1)
    per_sm = 1;
  const int64_t want = (int64_t)(sms > 0 ? sms : 1) * per_sm;
  return (int)(t.n_tiles < want ? t.n_tiles : want);
}

// The call's one device->host read: the first h.size() bytes of its out buffer, status word first; fails on a bad status.
static int read_back(const char* out, std::vector<char>& h, int n_labels, const char* who, cudaStream_t st) {
  DMN_CUDA(cudaMemcpyAsync(h.data(), out, h.size(), cudaMemcpyDeviceToHost, st));
  DMN_CUDA(cudaStreamSynchronize(st));
  int bad;
  memcpy(&bad, h.data(), sizeof(int));
  DMN_CHECK(!(bad & INV_BAD_NAN), "%s: the grid holds NaN values", who);
  DMN_CHECK(!(bad & INV_BAD_LABEL), "%s: the label grid holds a label outside [0, %d]", who, n_labels - 1);
  return 0;
}

int object_voxels(InventoryState& s, const float* occ, const int16_t* labels, int dim, float level, int n_labels,
                  const int32_t* boxes_host, int64_t* moments_host, uint32_t* hist_host, cudaStream_t st) {
  const char* who = "object_voxels";
  if (check_args(occ, dim, n_labels, who)) return 1;
  DMN_CHECK(moments_host != nullptr, "%s: moments is NULL", who);
  DMN_CHECK(!(level != level), "%s: level is NaN", who);
  const size_t mom_bytes = (size_t)n_labels * N_MOM * sizeof(uint64_t), hist_bytes = (size_t)n_labels * 3 * dim * sizeof(uint32_t);
  const size_t out_bytes = 16 + mom_bytes + hist_bytes;
  char* out;
  if (s.out.get(out_bytes, &out)) return 2;
  int* bad = reinterpret_cast<int*>(out);
  auto* mom = reinterpret_cast<unsigned long long*>(out + 16);
  auto* hist = reinterpret_cast<uint32_t*>(out + 16 + mom_bytes);
  int* boxes = nullptr;
  if (boxes_host) {
    if (s.in.get((size_t)n_labels * 6, &boxes)) return 2;
    DMN_CUDA(cudaMemcpyAsync(boxes, boxes_host, (size_t)n_labels * 6 * sizeof(int), cudaMemcpyHostToDevice, st));
  }
  DMN_CUDA(cudaMemsetAsync(out, 0, out_bytes, st));
  const InvTiling tl = tiling(dim);
  const size_t smem = (size_t)n_labels * (2 * TILE + 2) * sizeof(uint32_t) + (boxes ? (size_t)n_labels * 6 * sizeof(int) : 0);
  object_voxels_kernel<<<grid_blocks(tl, smem, (const void*)object_voxels_kernel), THREADS, smem, st>>>(
      occ, labels, tl, level, n_labels, boxes, mom, hist, bad);
  DMN_LAUNCH_OK();
  std::vector<char> h(out_bytes);
  if (const int rc = read_back(out, h, n_labels, who, st)) return rc;
  memcpy(moments_host, h.data() + 16, mom_bytes);
  if (hist_host) memcpy(hist_host, h.data() + 16 + mom_bytes, hist_bytes);
  return 0;
}

int object_spans(InventoryState& s, const float* occ, const int16_t* labels, int dim, float level, int n_labels,
                 const int32_t* boxes_host, const double* axes_host, double* spans_host, cudaStream_t st) {
  const char* who = "object_spans";
  if (check_args(occ, dim, n_labels, who)) return 1;
  DMN_CHECK(boxes_host && axes_host && spans_host, "%s: NULL boxes / axes / spans", who);
  DMN_CHECK(!(level != level), "%s: level is NaN", who);
  for (int q = 0; q < n_labels * 12; ++q)
    DMN_CHECK(std::isfinite(axes_host[q]), "%s: axis coefficient %d of label %d is not finite", who, q % 12, q / 12);
  const size_t key_bytes = (size_t)n_labels * 6 * sizeof(long long), out_bytes = 16 + key_bytes;
  const size_t axes_bytes = (size_t)n_labels * 12 * sizeof(double), box_bytes = (size_t)n_labels * 6 * sizeof(int);
  char *out, *in_d;
  if (s.out.get(out_bytes, &out) || s.in.get(axes_bytes + box_bytes, &in_d)) return 2;
  // inputs and the empty extrema go up in one copy each: [status | keys] and [axes | boxes]
  std::vector<char> init(out_bytes, 0);
  for (int q = 0; q < n_labels * 6; ++q) {
    const long long k0 = (q & 1) ? (long long)0x800fffffffffffffULL : 0x7ff0000000000000LL;
    memcpy(init.data() + 16 + q * sizeof(long long), &k0, sizeof(k0));
  }
  std::vector<char> in(axes_bytes + box_bytes);
  memcpy(in.data(), axes_host, axes_bytes);
  memcpy(in.data() + axes_bytes, boxes_host, box_bytes);
  DMN_CUDA(cudaMemcpyAsync(out, init.data(), out_bytes, cudaMemcpyHostToDevice, st));
  DMN_CUDA(cudaMemcpyAsync(in_d, in.data(), in.size(), cudaMemcpyHostToDevice, st));
  int* bad = reinterpret_cast<int*>(out);
  auto* keys = reinterpret_cast<long long*>(out + 16);
  const auto* axes = reinterpret_cast<const double*>(in_d);
  const auto* boxes = reinterpret_cast<const int*>(in_d + axes_bytes);
  const InvTiling tl = tiling(dim);
  const size_t smem = key_bytes + (size_t)n_labels * sizeof(int) + box_bytes;
  object_spans_kernel<<<grid_blocks(tl, smem, (const void*)object_spans_kernel), THREADS, smem, st>>>(
      occ, labels, tl, level, n_labels, boxes, axes, keys, bad);
  DMN_LAUNCH_OK();
  std::vector<char> h(out_bytes);
  if (const int rc = read_back(out, h, n_labels, who, st)) return rc;
  for (int q = 0; q < n_labels * 6; ++q) {
    long long key;
    memcpy(&key, h.data() + 16 + q * sizeof(long long), sizeof(key));
    spans_host[q] = key_value(key);
  }
  return 0;
}

}  // namespace dmnerf
