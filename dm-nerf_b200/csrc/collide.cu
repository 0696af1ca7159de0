// Collision checks for object moves (DESIGN.md, "Collision checks"): grid-only passes over a labelled keep-all sweep.
//   move_overlap:    per candidate move, the grid points the moved object covers after the move (landed) and, per label, those
//                    of them that hold a solid obstacle point (overlap).  The moved object at p is the unedited grid at the nearest
//                    grid index of the move's target t = trans p, exactly as the edited sweep samples it (edit_target).
//   object_contacts: per index axis a and label pair, the solid points of one label whose +a neighbour is a solid point of another.
// Every count is an integer (shared-memory histograms flushed with integer atomics), so the results do not depend on the launch
// shape or on the order of the atomics.  The network is not evaluated.
#include <cmath>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "ray_ops.cuh"
#include "sweep_grid.cuh"

namespace dmnerf {

namespace {

constexpr int RUN = 8;                        // candidates a block walks for each destination point it reads
constexpr int OV_THREADS = 256;
constexpr int OV_POINTS = 4;                  // destination points per thread
constexpr int OV_BLOCK_POINTS = OV_THREADS * OV_POINTS;
constexpr int N_COUNTERS = DMNERF_MAX_INS + 2;   // overlap per label 0 .. 127, then landed
constexpr int LANDED = DMNERF_MAX_INS + 1;
constexpr int CT_THREADS = 512;
constexpr int GE_THREADS = 256;
constexpr unsigned FULL = 0xffffffffu;

enum { BAD_NAN = 1, BAD_LABEL = 2 };

// One checked candidate as the kernel reads it: the move, its source box B and its destination box D (every point p with
// src(p) lies in D; an axis with dlo > dhi: none).
struct Candidate {
  double trans[12];
  double lo[3], hi[3];
  int dlo[3], dhi[3];
  Region piece;                 // bits NULL: the whole label moves
  ObjMask group;                // the labels that move together
  int label, rest_drop;
};

// A run of up to RUN consecutive candidates: the box holding their destination boxes, and the first block that works on it.
struct Run {
  int first, count;
  int lo[3], n[3];
  int64_t block0;
};

struct IndexMap {
  double inv[9], b[3];
};

__global__ void grid_check_kernel(const float* __restrict__ occ, const int16_t* __restrict__ labels, int64_t n, int n_labels,
                                  int* bad) {
  int flags = 0;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
    const float v = occ[p];
    const int l = labels[p];
    if (v != v) flags |= BAD_NAN;
    if (l < 0 || l >= n_labels) flags |= BAD_LABEL;
  }
  flags = __reduce_or_sync(FULL, flags);
  if ((threadIdx.x & 31) == 0 && flags) atomicOr(bad, flags);
}

// COPY (DESIGN.md, "Copying objects"): every candidate of the launch is a copy, which vacates nothing, so its own label's solid
// points are obstacles like any other.  DEFORM (DESIGN.md, "Deforming objects"): the candidates' targets are pulled through their
// deformations defs [n] (one per candidate row; n_knots 0: rigid).
template <bool COPY, bool DEFORM>
__global__ void __launch_bounds__(OV_THREADS) move_overlap_kernel(const GridXform g, const IndexMap map, const float* __restrict__ occ,
                                                                  const int16_t* __restrict__ labels, float level, ObjMask obstacles,
                                                                  const Candidate* __restrict__ cands, const Run* __restrict__ runs,
                                                                  int n_runs, unsigned long long* __restrict__ counts,
                                                                  const Deform* __restrict__ defs) {
  __shared__ Candidate sc[RUN];
  __shared__ uint32_t hist[RUN][N_COUNTERS];
  __shared__ int s_run;
  if (threadIdx.x == 0) {                                        // the run of this block: the last with block0 <= blockIdx.x
    int lo = 0, hi = n_runs - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (runs[mid].block0 <= (int64_t)blockIdx.x) lo = mid;
      else hi = mid - 1;
    }
    s_run = lo;
  }
  for (int q = threadIdx.x; q < RUN * N_COUNTERS; q += OV_THREADS) (&hist[0][0])[q] = 0;
  __syncthreads();
  const Run run = runs[s_run];
  {
    const int words = run.count * (int)(sizeof(Candidate) / sizeof(int));
    const int* src = reinterpret_cast<const int*>(cands + run.first);
    for (int q = threadIdx.x; q < words; q += OV_THREADS) reinterpret_cast<int*>(sc)[q] = src[q];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t d = g.dim;
  const int64_t plane = (int64_t)run.n[1] * run.n[2], volume = plane * run.n[0];
  const int64_t first = ((int64_t)blockIdx.x - run.block0) * OV_BLOCK_POINTS;
  for (int r = 0; r < OV_POINTS; ++r) {
    const int64_t w = first + (int64_t)r * OV_THREADS + threadIdx.x;
    const bool valid = w < volume;                               // not warp-uniform: the ballots below take every lane
    int idx[3] = {0, 0, 0};
    float p[3] = {0.f, 0.f, 0.f};
    int l = -1;
    bool solid = false;
    if (valid) {
      idx[0] = run.lo[0] + (int)(w / plane);
      idx[1] = run.lo[1] + (int)((w / run.n[2]) % run.n[1]);
      idx[2] = run.lo[2] + (int)(w % run.n[2]);
      const int64_t lin = ((int64_t)idx[0] * d + idx[1]) * d + idx[2];
      l = labels[lin];
      solid = occ[lin] > level && l >= 0 && l <= DMNERF_MAX_INS;
      sweep_point(g, lin, p);
    }
    const bool blocking = solid && obj_kept(obstacles, l);     // before the move's own vacating
    for (int c = 0; c < run.count; ++c) {
      const Candidate& m = sc[c];
      bool src = valid;
#pragma unroll
      for (int a = 0; a < 3; ++a) src = src && idx[a] >= m.dlo[a] && idx[a] <= m.dhi[a];
      float t[3];
      if (src) {
        double q[3];
        if (DEFORM && defs[run.first + c].n_knots) {
          src = true;
          edit_target_deformed(m.trans, defs[run.first + c], map.inv, map.b, m.lo, m.hi, src, p, t, q);
        } else {
          src = edit_target(m.trans, map.inv, map.b, m.lo, m.hi, true, p, t, q);
        }
        if (src) {
          const int64_t qi = ((int64_t)q[0] * d + (int64_t)q[1]) * d + (int64_t)q[2];
          const int lq = labels[qi];
          src = in_group(m.group, lq) && occ[qi] > level && (m.piece.bits == nullptr || !region_drops(m.piece, lq, t[0], t[1], t[2]));
        }
      }
      const unsigned landed = __ballot_sync(FULL, src);
      if (lane == 0 && landed) atomicAdd(&hist[c][LANDED], (uint32_t)__popc(landed));
      bool hit = src && blocking;
      if (!COPY && hit && in_group(m.group, l))                  // a point the move vacates is no obstacle
        hit = !(m.rest_drop || m.piece.bits == nullptr || !region_drops(m.piece, l, p[0], p[1], p[2]));
      if (hit) atomicAdd(&hist[c][l], 1u);
    }
  }
  __syncthreads();
  for (int q = threadIdx.x; q < run.count * N_COUNTERS; q += OV_THREADS) {
    const uint32_t v = (&hist[0][0])[q];
    if (v) atomicAdd(counts + (int64_t)run.first * N_COUNTERS + q, (unsigned long long)v);
  }
}

// One move of the grid-only edit (DESIGN.md, "Arranging objects"), one thread per grid point p of the state: edit_rule with the
// source grid at the target's nearest index q.  counts [129]: overwritten per label, then landed -- the takes whose target is
// solid, and those of them that land on a solid state point the move does not vacate, by its label.  The state point is read
// before it is written and no thread reads another's point, so the launch order of the points does not matter.  A COPY takes and
// never vacates, so every solid state point it lands on counts, its own label's included.  DEFORM: the target is pulled through
// the deformation df (edit_target_deformed).
template <bool COPY, bool DEFORM>
__global__ void __launch_bounds__(GE_THREADS) grid_edit_kernel(const GridXform g, const EditMove e, const float* __restrict__ src_occ,
                                                               const int16_t* __restrict__ src_labels, float level,
                                                               float* __restrict__ occ, int16_t* __restrict__ labels,
                                                               unsigned long long* __restrict__ counts, const Deform df) {
  __shared__ uint32_t hist[N_COUNTERS];
  for (int k = threadIdx.x; k < N_COUNTERS; k += GE_THREADS) hist[k] = 0;
  __syncthreads();
  const int64_t d = g.dim, p = (int64_t)blockIdx.x * GE_THREADS + threadIdx.x;
  bool landed = false;
  if (p < d * d * d) {
    const float o = occ[p];
    const int l = labels[p];
    float x[3], t[3];
    double q[3];
    sweep_point(g, p, x);
    bool in_box = !e.empty;
    if (DEFORM)
      edit_target_deformed(e.trans, df, e.inv, e.b, e.lo, e.hi, in_box, x, t, q);
    else
      in_box = edit_target(e.trans, e.inv, e.b, e.lo, e.hi, in_box, x, t, q);
    auto here = [&](int lp) { return e.piece.bits == nullptr || !region_drops(e.piece, lp, x[0], x[1], x[2]); };
    edit_rule<COPY>(
        e, in_box,
        [&](int& lt, float& ot) {
          const int64_t qi = ((int64_t)q[0] * d + (int64_t)q[1]) * d + (int64_t)q[2];
          lt = src_labels[qi];
          ot = src_occ[qi];
        },
        o, l, level, [&](int lt) { return region_drops(e.piece, lt, t[0], t[1], t[2]); }, [&](bool& b, int lp) { b = here(lp); },
        [&](float ot, int lt) {
          occ[p] = ot;
          labels[p] = (int16_t)lt;
          landed = ot > level;
          if (landed && o > level && (COPY || !(in_group(e.group, l) && (e.rest_drop || here(l))))) atomicAdd(&hist[l], 1u);
        },
        [&] { occ[p] = 0.0f; });
  }
  const unsigned n = __ballot_sync(FULL, landed);
  if ((threadIdx.x & 31) == 0 && n) atomicAdd(&hist[LANDED], (uint32_t)__popc(n));
  __syncthreads();
  for (int k = threadIdx.x; k < N_COUNTERS; k += GE_THREADS)
    if (hist[k]) atomicAdd(counts + k, (unsigned long long)hist[k]);
}

// shared: faces [3][n_labels][n_labels]; a block walks points p grid-stride and counts the +a neighbours of its solid points
__global__ void __launch_bounds__(CT_THREADS) object_contacts_kernel(const float* __restrict__ occ, const int16_t* __restrict__ labels,
                                                                     int dim, float level, int n_labels,
                                                                     unsigned long long* __restrict__ faces, int* bad) {
  extern __shared__ uint32_t sf[];
  const int nn = n_labels * n_labels;
  for (int q = threadIdx.x; q < 3 * nn; q += CT_THREADS) sf[q] = 0;
  __syncthreads();
  const int64_t d = dim, n = d * d * d;
  const int64_t stride[3] = {d * d, d, 1};
  int flags = 0;
  for (int64_t p = (int64_t)blockIdx.x * CT_THREADS + threadIdx.x; p < n; p += (int64_t)gridDim.x * CT_THREADS) {
    const float v = occ[p];
    const int l = labels[p];
    if (v != v) flags |= BAD_NAN;
    if (l < 0 || l >= n_labels) {
      flags |= BAD_LABEL;
      continue;
    }
    if (!(v > level)) continue;
    const int idx[3] = {(int)(p / (d * d)), (int)((p / d) % d), (int)(p % d)};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (idx[a] + 1 >= dim) continue;                           // never across a grid face
      const int64_t q = p + stride[a];
      const int l2 = labels[q];
      if (l2 != l && l2 >= 0 && l2 < n_labels && occ[q] > level) atomicAdd(sf + (a * n_labels + l) * n_labels + l2, 1u);
    }
  }
  flags = __reduce_or_sync(FULL, flags);
  if ((threadIdx.x & 31) == 0 && flags) atomicOr(bad, flags);
  __syncthreads();
  for (int q = threadIdx.x; q < 3 * nn; q += CT_THREADS)
    if (sf[q]) atomicAdd(faces + q, (unsigned long long)sf[q]);
}

int persistent_blocks(const void* kernel, int threads, size_t smem, int64_t min_blocks) {
  int dev = 0, sms = 0, per_sm = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem) != cudaSuccess || per_sm < 1)
    per_sm = 1;
  const int64_t want = (int64_t)(sms > 0 ? sms : 1) * per_sm;
  return (int)(want > min_blocks ? want : min_blocks);
}

// The call's one device->host read: status word, then the counters; fails on a bad status.
int read_back(const char* out, std::vector<char>& h, int max_label, const char* who, cudaStream_t st) {
  return read_checked(out, h.data(), h.size(), max_label, who, st);
}

// The grid's index map forward, x = A u + b (objects.grid_affine): A = S R diag(extents / (dim - 1)), S: (x, y, z) -> (x, -z, y).
void grid_forward(const double* T, const double* ext, int dim, double A[9]) {
  const double R[3][3] = {{T[0], T[1], T[2]}, {T[4], T[5], T[6]}, {T[8], T[9], T[10]}};
  const double SR[3][3] = {{R[0][0], R[0][1], R[0][2]}, {-R[2][0], -R[2][1], -R[2][2]}, {R[1][0], R[1][1], R[1][2]}};
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) A[3 * r + c] = SR[r][c] * (ext[c] / (double)(dim - 1));
}

// The forward image D(s) of a network-frame point s under the deformation d (DESIGN.md, "Deforming objects"), its frame
// coordinates given: (u, v) -> A(h) (u, v) + t(h), h kept, the table clamped to the end knots.
static void deform_forward(const dmnerf_deformation& d, double u, double v, double h, double out[3]) {
  const int K = d.n_knots;
  const double r = (h - d.h0) / d.dh;
  const double kf = std::fmin(std::fmax(std::floor(r), 0.0), (double)(K - 2));
  const double s = std::fmin(std::fmax(r - kf, 0.0), 1.0);
  const double* k0 = d.knots + 6 * (int)kf;
  double a[6];
  for (int j = 0; j < 6; ++j) a[j] = k0[j] + s * (k0[6 + j] - k0[j]);
  const double uu = a[0] * u + a[1] * v + a[4], vv = a[2] * u + a[3] * v + a[5];
  for (int c = 0; c < 3; ++c) out[c] = d.frame[9 + c] + uu * d.frame[c] + vv * d.frame[3 + c] + h * d.frame[6 + c];
}

// The destination box of a move with source box B (DESIGN.md, "Collision checks", destination culling): B grown by half a voxel,
// its 8 corners mapped by idx_p = inv (M^-1 (A u + b - m) - b), floor / ceil, one voxel of margin, clipped to the grid.  A
// non-finite corner (a nearly degenerate move) keeps the whole grid.  A deformed move (def, n_knots > 0; DESIGN.md, "Deforming
// objects") maps D(B) instead: B bounded in frame coordinates as [u] x [v] x [h], and the images of that box's 4 horizontal
// corners at its two heights and at every knot height between them, which hold D(B) because D is affine in (u, v) and, within a
// knot interval, in h.
void destination_box(const EditMove& e, const double A[9], int dim, const dmnerf_deformation* def, int dlo[3], int dhi[3]) {
  const double* t = e.trans;
  const double M[3][3] = {{t[0], t[1], t[2]}, {t[4], t[5], t[6]}, {t[8], t[9], t[10]}};
  double Mi[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      const int i1 = (j + 1) % 3, i2 = (j + 2) % 3, j1 = (i + 1) % 3, j2 = (i + 2) % 3;
      Mi[i][j] = M[i1][j1] * M[i2][j2] - M[i1][j2] * M[i2][j1];
    }
  const double det = M[0][0] * Mi[0][0] + M[0][1] * Mi[1][0] + M[0][2] * Mi[2][0];
  double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  bool finite = true;
  auto add = [&](const double s[3]) {                            // a source point s of the network frame
    double x[3], y[3];
    for (int r = 0; r < 3; ++r) x[r] = s[r] - t[4 * r + 3];
    for (int r = 0; r < 3; ++r) y[r] = (Mi[r][0] * x[0] + Mi[r][1] * x[1] + Mi[r][2] * x[2]) / det - e.b[r];
    for (int a = 0; a < 3; ++a) {
      const double v = e.inv[3 * a] * y[0] + e.inv[3 * a + 1] * y[1] + e.inv[3 * a + 2] * y[2];
      finite = finite && std::isfinite(v);
      lo[a] = v < lo[a] ? v : lo[a];
      hi[a] = v > hi[a] ? v : hi[a];
    }
  };
  const bool deformed = def && def->n_knots;
  double flo[3] = {INFINITY, INFINITY, INFINITY}, fhi[3] = {-INFINITY, -INFINITY, -INFINITY};   // B in frame coordinates
  for (int c = 0; c < 8; ++c) {
    double u[3], s[3];
    for (int a = 0; a < 3; ++a) u[a] = (c >> a) & 1 ? e.hi[a] + 0.5 : e.lo[a] - 0.5;
    for (int r = 0; r < 3; ++r) s[r] = A[3 * r] * u[0] + A[3 * r + 1] * u[1] + A[3 * r + 2] * u[2] + e.b[r];
    if (!deformed) {
      add(s);
      continue;
    }
    for (int a = 0; a < 3; ++a) {
      const double* ax = def->frame + 3 * a;
      const double f = ax[0] * (s[0] - def->frame[9]) + ax[1] * (s[1] - def->frame[10]) + ax[2] * (s[2] - def->frame[11]);
      flo[a] = f < flo[a] ? f : flo[a];
      fhi[a] = f > fhi[a] ? f : fhi[a];
    }
  }
  if (deformed) {
    auto level = [&](double h) {
      for (int c = 0; c < 4; ++c) {
        double s[3];
        deform_forward(*def, c & 1 ? fhi[0] : flo[0], c & 2 ? fhi[1] : flo[1], h, s);
        add(s);
      }
    };
    level(flo[2]);
    level(fhi[2]);
    for (int k = 0; k < def->n_knots; ++k) {
      const double h = def->h0 + k * def->dh;
      if (h > flo[2] && h < fhi[2]) level(h);
    }
  }
  for (int a = 0; a < 3; ++a) {
    const double l = finite ? std::floor(lo[a]) - 1.0 : 0.0, h = finite ? std::ceil(hi[a]) + 1.0 : (double)(dim - 1);
    dlo[a] = l < 0.0 ? 0 : (l > dim - 1 ? dim : (int)l);                  // dim: the box misses the grid
    dhi[a] = h > dim - 1 ? dim - 1 : (h < 0.0 ? -1 : (int)h);
  }
}

}  // namespace

int launch_grid_check(const float* occ, const int16_t* labels, int64_t n, int n_labels, int* bad, cudaStream_t st) {
  grid_check_kernel<<<persistent_blocks((const void*)grid_check_kernel, 256, 0, 1), 256, 0, st>>>(occ, labels, n, n_labels, bad);
  DMN_LAUNCH_OK();
  return 0;
}

int read_checked(const void* dev, void* host, size_t bytes, int max_label, const char* who, cudaStream_t st) {
  DMN_CUDA(cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, st));
  DMN_CUDA(cudaStreamSynchronize(st));
  int bad;
  memcpy(&bad, host, sizeof(int));
  DMN_CHECK(!(bad & BAD_NAN), "%s: the grid holds NaN values", who);
  DMN_CHECK(!(bad & BAD_LABEL), "%s: the label grid holds a label outside [0, %d]", who, max_label);
  return 0;
}

int move_overlap(InventoryState& s, const float* occ, const int16_t* labels, int dim, float level, const double* T16, const double* ext3,
                 const dmnerf_edit_move* cands_host, const int32_t* copies_host, const uint32_t* groups_host, int n,
                 const uint32_t* obstacles_host, int64_t* overlap_host, int64_t* landed_host, cudaStream_t st, const char* who,
                 const dmnerf_deformation* deformations_host) {
  if (deformations_check(deformations_host, n > 0 ? n : 0, who)) return 1;
  DMN_CHECK(occ && labels && T16 && ext3 && overlap_host && landed_host, "%s: NULL argument", who);
  if (sweep_grid_check(T16, ext3, dim, level, who)) return 1;
  DMN_CHECK(n >= 1 && n <= DMNERF_MAX_CANDIDATES, "%s: between 1 and %d candidates are supported, got %d", who,
            DMNERF_MAX_CANDIDATES, n);
  DMN_CHECK(cands_host, "%s: candidates is NULL", who);
  if (copy_flags_check(cands_host, copies_host, groups_host, n, false, who)) return 1;   // each candidate on its own: no order
  // the moves first, then the copies: one launch per kind, slot[i] the row of candidate i
  std::vector<int> slot(n);
  int n_moves = 0;
  for (int i = 0; i < n; ++i)
    if (!copies_host || !copies_host[i]) slot[i] = n_moves++;
  for (int i = 0, k = n_moves; i < n; ++i)
    if (copies_host && copies_host[i]) slot[i] = k++;
  std::vector<Candidate> cand(n);
  double A[9];
  grid_forward(T16, ext3, dim, A);
  IndexMap map{};
  for (int i = 0; i < n; ++i) {
    EditMove e;
    if (edit_move_from_abi(cands_host[i], T16, ext3, dim, DMNERF_MAX_INS, e, who, i, groups_host ? groups_host + 4 * i : nullptr))
      return 1;
    if (i == 0) {
      memcpy(map.inv, e.inv, sizeof(map.inv));
      memcpy(map.b, e.b, sizeof(map.b));
    }
    Candidate& c = cand[slot[i]];
    memset(&c, 0, sizeof(c));
    memcpy(c.trans, e.trans, sizeof(c.trans));
    memcpy(c.lo, e.lo, sizeof(c.lo));
    memcpy(c.hi, e.hi, sizeof(c.hi));
    if (e.empty) {
      for (int a = 0; a < 3; ++a) { c.dlo[a] = 1; c.dhi[a] = 0; }
    } else {
      destination_box(e, A, dim, deformations_host ? deformations_host + i : nullptr, c.dlo, c.dhi);
    }
    c.piece = e.piece;
    c.group = e.group;
    c.label = e.label;
    c.rest_drop = e.rest_drop;
  }
  ObjMask obst;
  for (int w = 0; w < 4; ++w) obst.w[w] = obstacles_host ? obstacles_host[w] : 0xffffffffu;
  // per kind (moves, then copies), runs of RUN consecutive candidates over the box holding their destination boxes, each kind's
  // blocks counted from 0 for its own launch
  std::vector<Run> runs;
  int64_t blocks_of[2] = {0, 0};
  size_t first_run[3] = {0, 0, 0};
  for (int kind = 0; kind < 2; ++kind) {
    const int begin = kind ? n_moves : 0, end = kind ? n : n_moves;
    for (int f = begin; f < end; f += RUN) {
      Run r{};
      r.first = f;
      r.count = end - f < RUN ? end - f : RUN;
      int lo[3] = {dim, dim, dim}, hi[3] = {-1, -1, -1};
      for (int i = f; i < f + r.count; ++i) {
        const Candidate& c = cand[i];
        if (c.dlo[0] > c.dhi[0] || c.dlo[1] > c.dhi[1] || c.dlo[2] > c.dhi[2]) continue;
        for (int a = 0; a < 3; ++a) {
          lo[a] = c.dlo[a] < lo[a] ? c.dlo[a] : lo[a];
          hi[a] = c.dhi[a] > hi[a] ? c.dhi[a] : hi[a];
        }
      }
      if (hi[0] < 0) continue;                                   // no candidate of the run reaches the grid
      int64_t volume = 1;
      for (int a = 0; a < 3; ++a) {
        r.lo[a] = lo[a];
        r.n[a] = hi[a] - lo[a] + 1;
        volume *= r.n[a];
      }
      r.block0 = blocks_of[kind];
      blocks_of[kind] += (volume + OV_BLOCK_POINTS - 1) / OV_BLOCK_POINTS;
      runs.push_back(r);
    }
    first_run[kind + 1] = runs.size();
    DMN_CHECK(blocks_of[kind] < INT32_MAX, "%s: %lld blocks of work exceed one launch", who, (long long)blocks_of[kind]);
  }
  const size_t count_bytes = (size_t)n * N_COUNTERS * sizeof(unsigned long long), out_bytes = 16 + count_bytes;
  const size_t cand_bytes = (size_t)n * sizeof(Candidate), run_bytes = runs.size() * sizeof(Run);
  // the deformations in candidate rows, after the runs (none: no bytes)
  std::vector<Deform> defs(n), def_rows;
  bool deformed = false;
  if (deformations_from_abi(deformations_host, n, s.knots, defs.data(), &deformed, who, st)) return 1;
  if (deformed) {
    def_rows.resize(n);
    for (int i = 0; i < n; ++i) def_rows[slot[i]] = defs[i];
  }
  const size_t def_bytes = def_rows.size() * sizeof(Deform);
  char *out, *in_d;
  if (s.out.get(out_bytes, &out) || s.in.get(cand_bytes + run_bytes + def_bytes + 16, &in_d)) return 2;
  const size_t def_at = (cand_bytes + run_bytes + 15) / 16 * 16;
  std::vector<char> in(def_at + def_bytes);
  memcpy(in.data(), cand.data(), cand_bytes);
  if (run_bytes) memcpy(in.data() + cand_bytes, runs.data(), run_bytes);
  if (def_bytes) memcpy(in.data() + def_at, def_rows.data(), def_bytes);
  const Deform* defs_d = deformed ? reinterpret_cast<const Deform*>(in_d + def_at) : nullptr;
  DMN_CUDA(cudaMemsetAsync(out, 0, out_bytes, st));
  DMN_CUDA(cudaMemcpyAsync(in_d, in.data(), in.size(), cudaMemcpyHostToDevice, st));
  int* bad = reinterpret_cast<int*>(out);
  auto* counts = reinterpret_cast<unsigned long long*>(out + 16);
  const int64_t npts = (int64_t)dim * dim * dim;
  if (launch_grid_check(occ, labels, npts, DMNERF_MAX_INS + 1, bad, st)) return 2;
  const GridXform g = make_xform(T16, ext3, dim);
  const Candidate* cands_d = reinterpret_cast<const Candidate*>(in_d);
  for (int kind = 0; kind < 2; ++kind) {
    if (!blocks_of[kind]) continue;
    const Run* runs_d = reinterpret_cast<const Run*>(in_d + cand_bytes) + first_run[kind];
    const int n_runs = (int)(first_run[kind + 1] - first_run[kind]);
    const unsigned nb = (unsigned)blocks_of[kind];
    if (kind && deformed)
      move_overlap_kernel<true, true><<<nb, OV_THREADS, 0, st>>>(g, map, occ, labels, level, obst, cands_d, runs_d, n_runs, counts,
                                                                 defs_d);
    else if (kind)
      move_overlap_kernel<true, false><<<nb, OV_THREADS, 0, st>>>(g, map, occ, labels, level, obst, cands_d, runs_d, n_runs, counts,
                                                                  nullptr);
    else if (deformed)
      move_overlap_kernel<false, true><<<nb, OV_THREADS, 0, st>>>(g, map, occ, labels, level, obst, cands_d, runs_d, n_runs, counts,
                                                                  defs_d);
    else
      move_overlap_kernel<false, false><<<nb, OV_THREADS, 0, st>>>(g, map, occ, labels, level, obst, cands_d, runs_d, n_runs, counts,
                                                                   nullptr);
    DMN_LAUNCH_OK();
  }
  std::vector<char> h(out_bytes);
  if (const int rc = read_back(out, h, DMNERF_MAX_INS, who, st)) return rc;
  for (int i = 0; i < n; ++i) {
    const char* row = h.data() + 16 + (size_t)slot[i] * N_COUNTERS * sizeof(unsigned long long);
    memcpy(overlap_host + (size_t)i * (DMNERF_MAX_INS + 1), row, (DMNERF_MAX_INS + 1) * sizeof(int64_t));
    memcpy(landed_host + i, row + LANDED * sizeof(int64_t), sizeof(int64_t));
  }
  return 0;
}

int object_contacts(InventoryState& s, const float* occ, const int16_t* labels, int dim, float level, int n_labels, int64_t* faces_host,
                    cudaStream_t st) {
  const char* who = "object_contacts";
  DMN_CHECK(occ && labels && faces_host, "%s: NULL argument", who);
  DMN_CHECK(dim >= 2 && dim <= 2048, "%s: dim %d out of range [2, 2048]", who, dim);
  DMN_CHECK(n_labels >= 1 && n_labels <= DMNERF_MAX_INS + 1, "%s: n_labels %d out of range [1, %d]", who, n_labels, DMNERF_MAX_INS + 1);
  DMN_CHECK(level > 0.0f && level < 1.0f, "%s: level %g outside (0, 1)", who, (double)level);
  const size_t nf = (size_t)3 * n_labels * n_labels, out_bytes = 16 + nf * sizeof(unsigned long long);
  char* out;
  if (s.out.get(out_bytes, &out)) return 2;
  DMN_CUDA(cudaMemsetAsync(out, 0, out_bytes, st));
  const size_t smem = nf * sizeof(uint32_t);
  DMN_CUDA(cudaFuncSetAttribute((const void*)object_contacts_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // a block's shared counters stay below 2^32: at most 3 per point it visits
  const int64_t npts = (int64_t)dim * dim * dim, min_blocks = (3 * npts) / ((int64_t)1 << 31) + 1;
  object_contacts_kernel<<<persistent_blocks((const void*)object_contacts_kernel, CT_THREADS, smem, min_blocks), CT_THREADS, smem, st>>>(
      occ, labels, dim, level, n_labels, reinterpret_cast<unsigned long long*>(out + 16), reinterpret_cast<int*>(out));
  DMN_LAUNCH_OK();
  std::vector<char> h(out_bytes);
  if (const int rc = read_back(out, h, n_labels - 1, who, st)) return rc;
  memcpy(faces_host, h.data() + 16, nf * sizeof(int64_t));
  return 0;
}

int grid_edit(InventoryState& s, const float* src_occ, const int16_t* src_labels, int dim, float level, const double* T16,
              const double* ext3, const dmnerf_edit_move* moves_host, const int32_t* copies_host, const uint32_t* groups_host, int n,
              float* occ, int16_t* labels, int64_t* landed_host, int64_t* overwritten_host, cudaStream_t st, const char* who,
              const dmnerf_deformation* deformations_host) {
  if (deformations_check(deformations_host, n > 0 ? n : 0, who)) return 1;
  DMN_CHECK(src_occ && src_labels && occ && labels && T16 && ext3 && landed_host && overwritten_host, "%s: NULL argument", who);
  DMN_CHECK(n >= 1 && n <= DMNERF_MAX_MOVES, "%s: between 1 and %d moves are supported, got %d", who, DMNERF_MAX_MOVES, n);
  DMN_CHECK(moves_host, "%s: moves is NULL", who);
  if (sweep_grid_check(T16, ext3, dim, level, who)) return 1;
  const int64_t npts = (int64_t)dim * dim * dim;
  // the state is written while the source is read at other points: they must not share memory
  auto apart = [](const void* a, size_t na, const void* b, size_t nb) {
    const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
    return x + na <= y || y + nb <= x;
  };
  const size_t fo = (size_t)npts * sizeof(float), lb = (size_t)npts * sizeof(int16_t);
  DMN_CHECK(apart(src_occ, fo, occ, fo) && apart(src_occ, fo, labels, lb) && apart(src_labels, lb, occ, fo) &&
                apart(src_labels, lb, labels, lb),
            "%s: the source and state grids overlap in memory (the state must be a separate copy)", who);
  std::vector<EditMove> mv(n);
  for (int i = 0; i < n; ++i)
    if (edit_move_from_abi(moves_host[i], T16, ext3, dim, DMNERF_MAX_INS, mv[i], who, i, groups_host ? groups_host + 4 * i : nullptr))
      return 1;
  if (copy_flags_check(moves_host, copies_host, groups_host, n, true, who)) return 1;
  std::vector<Deform> defs(n);
  if (deformations_from_abi(deformations_host, n, s.knots, defs.data(), nullptr, who, st)) return 1;
  const size_t out_bytes = 16 + (size_t)n * N_COUNTERS * sizeof(unsigned long long);
  char* out;
  if (s.out.get(out_bytes, &out)) return 2;
  DMN_CUDA(cudaMemsetAsync(out, 0, out_bytes, st));
  int* bad = reinterpret_cast<int*>(out);
  if (launch_grid_check(src_occ, src_labels, npts, DMNERF_MAX_INS + 1, bad, st) ||
      launch_grid_check(occ, labels, npts, DMNERF_MAX_INS + 1, bad, st))
    return 2;
  std::vector<char> h(out_bytes);
  if (const int rc = read_checked(out, h.data(), 16, DMNERF_MAX_INS, who, st)) return rc;   // a bad grid writes nothing
  const GridXform g = make_xform(T16, ext3, dim);
  auto* counts = reinterpret_cast<unsigned long long*>(out + 16);
  const unsigned ge_blocks = (unsigned)((npts + GE_THREADS - 1) / GE_THREADS);
  for (int i = 0; i < n; ++i) {
    unsigned long long* row = counts + (size_t)i * N_COUNTERS;
    const bool copy = copies_host && copies_host[i], deformed = defs[i].n_knots != 0;
    if (copy && deformed)
      grid_edit_kernel<true, true><<<ge_blocks, GE_THREADS, 0, st>>>(g, mv[i], src_occ, src_labels, level, occ, labels, row, defs[i]);
    else if (copy)
      grid_edit_kernel<true, false><<<ge_blocks, GE_THREADS, 0, st>>>(g, mv[i], src_occ, src_labels, level, occ, labels, row, defs[i]);
    else if (deformed)
      grid_edit_kernel<false, true><<<ge_blocks, GE_THREADS, 0, st>>>(g, mv[i], src_occ, src_labels, level, occ, labels, row, defs[i]);
    else
      grid_edit_kernel<false, false><<<ge_blocks, GE_THREADS, 0, st>>>(g, mv[i], src_occ, src_labels, level, occ, labels, row,
                                                                       defs[i]);
    DMN_LAUNCH_OK();
  }
  if (const int rc = read_back(out, h, DMNERF_MAX_INS, who, st)) return rc;
  for (int i = 0; i < n; ++i) {
    const char* row = h.data() + 16 + (size_t)i * N_COUNTERS * sizeof(unsigned long long);
    memcpy(overwritten_host + (size_t)i * (DMNERF_MAX_INS + 1), row, (DMNERF_MAX_INS + 1) * sizeof(int64_t));
    memcpy(landed_host + i, row + LANDED * sizeof(int64_t), sizeof(int64_t));
  }
  return 0;
}

}  // namespace dmnerf
