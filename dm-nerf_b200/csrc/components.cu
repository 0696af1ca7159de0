// Connected components (DESIGN.md, "Connected components") of the solid points (occ > level) of a grid [dim]^3, C order of
// the index (i, j, k), p = (i * dim + j) * dim + k.  Two solid points are adjacent when they are face neighbours
// (connectivity 6) or face, edge or corner neighbours (26) and, with a label grid, carry the same label; neighbours never wrap
// across a grid face.  A component's root is its smallest linear index; components are numbered 0 .. n - 1 in ascending root
// order.
//
// The parent array is the caller's id grid itself (int32, -1 = not solid), so no [dim]^3 scratch is allocated:
//   init:     parent[p] = the first point of p's run of adjacent points along k inside p's aligned group of 32 indices (a warp)
//   merge:    per solid point and backward neighbour, a lock-free union that hooks the larger root under the smaller one
//             (atomicCAS on roots only); parent[p] <= p always holds, so the final root is the component's minimum index
//   compress: parent[p] = root (atomicMin: every write is an ancestor, the root is the smallest)
//   number:   per chunk the root count, an exclusive scan, then the roots' ids in index order, written as -(id + 2)
//   resolve:  non-roots read their root's id; then the roots decode theirs.
// The result is a function of the grid alone: it does not depend on the launch shape or on the order of the atomics.
#include <cub/cub.cuh>

#include <cstring>

#include "common.cuh"

namespace dmnerf {

namespace {

constexpr int CC_THREADS = 256;
constexpr int CC_ITEMS = 8;                                  // consecutive points per thread of the numbering passes
constexpr int CC_CHUNK = CC_THREADS * CC_ITEMS;
constexpr int CC_MAX_DIM = 1290;                             // dim^3 < 2^31: int32 parents and ids
constexpr unsigned FULL = 0xffffffffu;

enum { CC_BAD_NAN = 1, CC_BAD_LABEL = 2, CC_BAD_ID = 4 };

__device__ __forceinline__ int64_t stride_of() { return (int64_t)gridDim.x * blockDim.x; }

// ---- init: solid points, validation, runs along k inside a warp ----------------------------------------------------------
__global__ void __launch_bounds__(CC_THREADS) cc_init_kernel(const float* __restrict__ occ, const int16_t* __restrict__ labels,
                                                             int64_t n, int dim, float level, int n_labels, int32_t* __restrict__ parent,
                                                             int* bad) {
  const int lane = threadIdx.x & 31;
  // the stride is a multiple of 32, so a warp always holds the aligned indices 32 q .. 32 q + 31
  for (int64_t base = (int64_t)blockIdx.x * CC_THREADS + (threadIdx.x & ~31); base < n; base += stride_of()) {
    const int64_t p = base + lane;
    bool solid = false;
    int lab = 0;
    if (p < n) {
      const float v = occ[p];
      lab = labels ? (int)labels[p] : 0;
      if (v != v) atomicOr(bad, CC_BAD_NAN);
      if (lab < 0 || lab >= n_labels) atomicOr(bad, CC_BAD_LABEL);
      else solid = v > level;
    }
    // joined to p - 1: both solid, one label, p not the first point of its row, p - 1 in this warp
    const int left_lab = __shfl_up_sync(FULL, lab, 1);
    const bool left_solid = __shfl_up_sync(FULL, solid, 1);
    const bool join = solid && lane > 0 && left_solid && left_lab == lab && (int)(p % dim) != 0;
    const unsigned starts = ~__ballot_sync(FULL, join);         // lanes that begin a run (or are not solid)
    const int first = 31 - __clz(starts & (0xffffffffu >> (31 - lane)));
    if (p < n) parent[p] = solid ? (int32_t)(base + first) : -1;
  }
}

// ---- merge ---------------------------------------------------------------------------------------------------------------
// find with path halving; only non-roots are written, and only with one of their ancestors
__device__ __forceinline__ int find_root(int32_t* parent, int x) {
  int cur = __ldcg(parent + x);
  if (cur == x) return x;
  int prev = x, next;
  while (cur > (next = __ldcg(parent + cur))) {
    parent[prev] = next;
    prev = cur;
    cur = next;
  }
  return cur;
}

__device__ __forceinline__ void unite(int32_t* parent, int a, int b) {
  a = find_root(parent, a);
  b = find_root(parent, b);
  while (a != b) {
    if (a > b) { const int t = a; a = b; b = t; }
    const int old = atomicCAS(parent + b, b, a);          // hook the larger root under the smaller
    if (old == b) return;
    b = find_root(parent, old);                            // b gained a parent meanwhile: retry from the roots
    a = find_root(parent, a);
  }
}

__device__ __forceinline__ bool joined(const int32_t* parent, const int16_t* labels, int64_t q, int lab) {
  return __ldcg(parent + q) >= 0 && (!labels || labels[q] == lab);
}

// The backward neighbours (di, dj, dk) < (0, 0, 0) lexicographically: 3 for connectivity 6, 13 for 26; (0, 0, -1) last.
__constant__ signed char c_back[13][3] = {{-1, -1, -1}, {-1, -1, 0}, {-1, -1, 1}, {-1, 0, -1}, {-1, 0, 0}, {-1, 0, 1}, {-1, 1, -1},
                                         {-1, 1, 0},   {-1, 1, 1},  {0, -1, -1}, {0, -1, 0},  {0, -1, 1}, {0, 0, -1}};
__constant__ signed char c_back6[3][3] = {{-1, 0, 0}, {0, -1, 0}, {0, 0, -1}};

template <int CONN>
__global__ void __launch_bounds__(CC_THREADS) cc_merge_kernel(const int16_t* __restrict__ labels, int64_t n, int dim,
                                                              int32_t* parent) {
  constexpr int NB = CONN == 6 ? 3 : 13;
  for (int64_t p = (int64_t)blockIdx.x * CC_THREADS + threadIdx.x; p < n; p += stride_of()) {
    if (__ldcg(parent + p) < 0) continue;
    const int lab = labels ? (int)labels[p] : 0;
    const int k = (int)(p % dim), j = (int)((p / dim) % dim), i = (int)(p / ((int64_t)dim * dim));
    const bool left = k > 0 && joined(parent, labels, p - 1, lab);
#pragma unroll
    for (int q = 0; q < NB - 1; ++q) {
      const int di = CONN == 6 ? c_back6[q][0] : c_back[q][0], dj = CONN == 6 ? c_back6[q][1] : c_back[q][1];
      const int dk = CONN == 6 ? c_back6[q][2] : c_back[q][2];
      const int ni = i + di, nj = j + dj, nk = k + dk;
      if (ni < 0 || nj < 0 || nj >= dim || nk < 0 || nk >= dim) continue;
      const int64_t r = p + ((int64_t)di * dim + dj) * dim + dk;
      if (!joined(parent, labels, r, lab)) continue;
      // p - 1 ~ p and r - 1 ~ r: thread p - 1 unites p - 1 with r - 1 along the same offset, which joins p and r
      if (left && nk > 0 && joined(parent, labels, r - 1, lab)) continue;
      unite(parent, (int)p, (int)r);
    }
    // (0, 0, -1): inside an aligned group of 32 the init already joined p to p - 1
    if (left && (p & 31) == 0) unite(parent, (int)p, (int)(p - 1));
  }
}

// ---- compress: every solid point points at its root ----------------------------------------------------------------------
__global__ void __launch_bounds__(CC_THREADS) cc_compress_kernel(int64_t n, int32_t* parent) {
  for (int64_t p = (int64_t)blockIdx.x * CC_THREADS + threadIdx.x; p < n; p += stride_of()) {
    int cur = __ldcg(parent + p);
    if (cur < 0 || cur == (int)p) continue;
    int prev = (int)p, next;
    while (cur > (next = __ldcg(parent + cur))) {
      atomicMin(parent + prev, next);
      prev = cur;
      cur = next;
    }
    atomicMin(parent + p, cur);
  }
}

// ---- numbering -----------------------------------------------------------------------------------------------------------
// chunk c = points c * CC_CHUNK .. (c + 1) * CC_CHUNK - 1, CC_ITEMS consecutive points per thread
__global__ void __launch_bounds__(CC_THREADS) cc_count_kernel(int64_t n, const int32_t* __restrict__ parent, int32_t* counts) {
  typedef cub::BlockReduce<int, CC_THREADS> Reduce;
  __shared__ typename Reduce::TempStorage tmp;
  const int64_t p0 = (int64_t)blockIdx.x * CC_CHUNK + (int64_t)threadIdx.x * CC_ITEMS;
  int c = 0;
#pragma unroll
  for (int q = 0; q < CC_ITEMS; ++q)
    if (p0 + q < n) c += parent[p0 + q] == (int)(p0 + q);
  const int total = Reduce(tmp).Sum(c);
  if (threadIdx.x == 0) counts[blockIdx.x] = total;
}

__global__ void __launch_bounds__(CC_THREADS) cc_number_roots_kernel(int64_t n, const int32_t* __restrict__ offsets, int32_t* parent) {
  typedef cub::BlockScan<int, CC_THREADS> Scan;
  __shared__ typename Scan::TempStorage tmp;
  const int64_t p0 = (int64_t)blockIdx.x * CC_CHUNK + (int64_t)threadIdx.x * CC_ITEMS;
  int c = 0;
#pragma unroll
  for (int q = 0; q < CC_ITEMS; ++q)
    if (p0 + q < n) c += parent[p0 + q] == (int)(p0 + q);
  int rank;
  Scan(tmp).ExclusiveSum(c, rank);
  int id = offsets[blockIdx.x] + rank;
#pragma unroll
  for (int q = 0; q < CC_ITEMS; ++q)
    if (p0 + q < n && parent[p0 + q] == (int)(p0 + q)) parent[p0 + q] = -(id++ + 2);
}

// non-roots (parent = root >= 0) take their root's id; the roots (<= -2) are only read here
__global__ void __launch_bounds__(CC_THREADS) cc_resolve_kernel(int64_t n, int32_t* parent) {
  for (int64_t p = (int64_t)blockIdx.x * CC_THREADS + threadIdx.x; p < n; p += stride_of()) {
    const int r = parent[p];
    if (r >= 0) parent[p] = -(parent[r] + 2);
  }
}

__global__ void __launch_bounds__(CC_THREADS) cc_decode_roots_kernel(int64_t n, int32_t* parent) {
  for (int64_t p = (int64_t)blockIdx.x * CC_THREADS + threadIdx.x; p < n; p += stride_of()) {
    const int r = parent[p];
    if (r <= -2) parent[p] = -(r + 2);
  }
}

// ---- per-component table and group map ----------------------------------------------------------------------------------
__global__ void __launch_bounds__(CC_THREADS) cc_table_kernel(const int32_t* __restrict__ comp, const int16_t* __restrict__ labels,
                                                              int64_t n, int64_t n_comp, int16_t* label, unsigned long long* voxels,
                                                              long long* root, int* bad) {
  const int lane = threadIdx.x & 31;
  for (int64_t base = (int64_t)blockIdx.x * CC_THREADS + (threadIdx.x & ~31); base < n; base += stride_of()) {
    const int64_t p = base + lane;
    int id = -1;
    if (p < n) {
      id = comp[p];
      if (id < -1 || id >= n_comp) {
        atomicOr(bad, CC_BAD_ID);
        id = -1;
      }
    }
    // lanes of one id: the lowest lane holds the smallest index
    const unsigned same = __match_any_sync(FULL, id);
    if (id >= 0 && lane == __ffs(same) - 1) {
      atomicAdd(voxels + id, (unsigned long long)__popc(same));
      atomicMin(root + id, (long long)p);
      label[id] = labels ? labels[p] : (int16_t)0;            // every point of a component carries its label
    }
  }
}

__global__ void __launch_bounds__(CC_THREADS) cc_groups_kernel(const int32_t* __restrict__ comp, int64_t n, int64_t n_comp,
                                                               const int16_t* __restrict__ lut, int16_t discard, int16_t* groups,
                                                               int* bad) {
  for (int64_t p = (int64_t)blockIdx.x * CC_THREADS + threadIdx.x; p < n; p += stride_of()) {
    const int id = comp[p];
    int16_t g = discard;
    if (id >= 0 && id < n_comp) g = lut[id];
    else if (id != -1) atomicOr(bad, CC_BAD_ID);
    groups[p] = g;
  }
}

int blocks_for(int64_t n) {
  const int64_t b = (n + CC_THREADS - 1) / CC_THREADS;
  const int64_t cap = 1 << 20;                                   // grid-stride beyond ~268 M points
  return (int)(b < cap ? b : cap);
}

int check_dim(int dim, const char* who) {
  DMN_CHECK(dim >= 2 && dim <= CC_MAX_DIM, "%s: dim %d out of range [2, %d] (dim^3 must stay below 2^31)", who, dim, CC_MAX_DIM);
  return 0;
}

}  // namespace

// the call's one device->host read: the status word and (object_components) the int32 total in the low half of the second word
static int read_status(const int64_t* status, int64_t* total_host, cudaStream_t st, const char* who, int n_labels) {
  int64_t h[2];
  DMN_CUDA(cudaMemcpyAsync(h, status, sizeof(h), cudaMemcpyDeviceToHost, st));
  DMN_CUDA(cudaStreamSynchronize(st));
  const int bad = (int)h[0];
  DMN_CHECK(!(bad & CC_BAD_NAN), "%s: the grid holds NaN values", who);
  DMN_CHECK(!(bad & CC_BAD_LABEL), "%s: the label grid holds a label outside [0, %d]", who, n_labels - 1);
  DMN_CHECK(!(bad & CC_BAD_ID), "%s: the id grid holds an id outside [-1, number of components)", who);
  if (total_host) *total_host = h[1];
  return 0;
}

int object_components(ComponentsState& s, const float* occ, const int16_t* labels, int dim, float level, int n_labels,
                      int connectivity, int32_t* comp, int64_t* n_components_host, cudaStream_t st) {
  const char* who = "object_components";
  DMN_CHECK(occ && comp && n_components_host, "%s: NULL occ / comp / n_components", who);
  if (check_dim(dim, who)) return 1;
  DMN_CHECK(n_labels >= 1 && n_labels <= DMNERF_MAX_INS + 1, "%s: n_labels %d out of range [1, %d]", who, n_labels, DMNERF_MAX_INS + 1);
  DMN_CHECK(connectivity == 6 || connectivity == 26, "%s: connectivity %d is not 6 or 26", who, connectivity);
  DMN_CHECK(!(level != level), "%s: level is NaN", who);
  const int64_t n = (int64_t)dim * dim * dim;
  const int64_t n_chunks = (n + CC_CHUNK - 1) / CC_CHUNK;
  int64_t* status;
  int32_t* counts;
  uint8_t* tmp;
  // status: [bad, total]; counts: n_chunks + 1 root counts (the last one 0), then their exclusive scan, the chunks' first ids
  // (its last entry is the total)
  if (s.status.get(2, &status) || s.counts.get((size_t)2 * (n_chunks + 1), &counts)) return 2;
  int32_t* offsets = counts + n_chunks + 1;
  size_t tmp_bytes = 0;
  DMN_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, counts, offsets, (int)(n_chunks + 1), st));
  if (s.temp.get(tmp_bytes, &tmp)) return 2;
  int* bad = reinterpret_cast<int*>(status);
  DMN_CUDA(cudaMemsetAsync(status, 0, 16, st));
  DMN_CUDA(cudaMemsetAsync(counts + n_chunks, 0, sizeof(int32_t), st));
  const int blocks = blocks_for(n);
  cc_init_kernel<<<blocks, CC_THREADS, 0, st>>>(occ, labels, n, dim, level, n_labels, comp, bad);
  DMN_LAUNCH_OK();
  if (connectivity == 6) cc_merge_kernel<6><<<blocks, CC_THREADS, 0, st>>>(labels, n, dim, comp);
  else cc_merge_kernel<26><<<blocks, CC_THREADS, 0, st>>>(labels, n, dim, comp);
  DMN_LAUNCH_OK();
  cc_compress_kernel<<<blocks, CC_THREADS, 0, st>>>(n, comp);
  DMN_LAUNCH_OK();
  cc_count_kernel<<<(unsigned)n_chunks, CC_THREADS, 0, st>>>(n, comp, counts);
  DMN_LAUNCH_OK();
  DMN_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, counts, offsets, (int)(n_chunks + 1), st));
  cc_number_roots_kernel<<<(unsigned)n_chunks, CC_THREADS, 0, st>>>(n, offsets, comp);
  DMN_LAUNCH_OK();
  cc_resolve_kernel<<<blocks, CC_THREADS, 0, st>>>(n, comp);
  DMN_LAUNCH_OK();
  cc_decode_roots_kernel<<<blocks, CC_THREADS, 0, st>>>(n, comp);
  DMN_LAUNCH_OK();
  // the total is offsets[n_chunks]: next to the status word, so that one read brings both
  DMN_CUDA(cudaMemcpyAsync(status + 1, offsets + n_chunks, sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  return read_status(status, n_components_host, st, who, n_labels);
}

int component_table(ComponentsState& s, const int32_t* comp, const int16_t* labels, int dim, int64_t n_comp, int16_t* label,
                    int64_t* voxels, int64_t* root, cudaStream_t st) {
  const char* who = "component_table";
  DMN_CHECK(comp != nullptr, "%s: comp is NULL", who);
  if (check_dim(dim, who)) return 1;
  const int64_t n = (int64_t)dim * dim * dim;
  DMN_CHECK(n_comp >= 0 && n_comp <= n, "%s: %lld components out of range [0, %lld]", who, (long long)n_comp, (long long)n);
  DMN_CHECK(n_comp == 0 || (label && voxels && root), "%s: NULL label / voxels / root", who);
  int64_t* status;
  if (s.status.get(2, &status)) return 2;
  DMN_CUDA(cudaMemsetAsync(status, 0, 16, st));
  if (n_comp) {
    DMN_CUDA(cudaMemsetAsync(voxels, 0, (size_t)n_comp * sizeof(int64_t), st));
    DMN_CUDA(cudaMemsetAsync(root, 0x7f, (size_t)n_comp * sizeof(int64_t), st));     // above every index: the empty minimum
  }
  cc_table_kernel<<<blocks_for(n), CC_THREADS, 0, st>>>(comp, labels, n, n_comp, label, reinterpret_cast<unsigned long long*>(voxels),
                                                        reinterpret_cast<long long*>(root), reinterpret_cast<int*>(status));
  DMN_LAUNCH_OK();
  return read_status(status, nullptr, st, who, 1);
}

int component_groups(ComponentsState& s, const int32_t* comp, int dim, int64_t n_comp, const int16_t* lut, int discard,
                     int16_t* groups, cudaStream_t st) {
  const char* who = "component_groups";
  DMN_CHECK(comp && groups, "%s: NULL comp / groups", who);
  if (check_dim(dim, who)) return 1;
  const int64_t n = (int64_t)dim * dim * dim;
  DMN_CHECK(n_comp >= 0 && n_comp <= n, "%s: %lld components out of range [0, %lld]", who, (long long)n_comp, (long long)n);
  DMN_CHECK(n_comp == 0 || lut, "%s: lut is NULL", who);
  DMN_CHECK(discard >= -32768 && discard <= 32767, "%s: discard group %d is not an int16", who, discard);
  int64_t* status;
  if (s.status.get(2, &status)) return 2;
  DMN_CUDA(cudaMemsetAsync(status, 0, 16, st));
  cc_groups_kernel<<<blocks_for(n), CC_THREADS, 0, st>>>(comp, n, n_comp, lut, (int16_t)discard, groups, reinterpret_cast<int*>(status));
  DMN_LAUNCH_OK();
  return read_status(status, nullptr, st, who, 1);
}

}  // namespace dmnerf
