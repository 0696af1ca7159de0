// Object placement (DESIGN.md, "Object placement"): where a lowered object comes to rest at every horizontal offset, from a
// labelled keep-all sweep, in index space and in integers.  Heights y run along the down axis, away from down; a column is one
// horizontal cell (h1, h2), numbered c = h1 dim + h2.
//   column pass: per column and height the highest obstacle height at or below it (int16, -1: none), each column contiguous, and
//                one byte per (column, height) that says whether the point belongs to the placed object;
//   runs:        per column the maximal vertical runs of the object, written in (column, bottom) order at the exclusive scan of
//                the per-column run counts, so that no atomic decides the order;
//   map:         one warp per offset: the free fall (warp minimum) and blocked (OR) over the runs, then the runs that rest on an
//                obstacle and a 128-bin shared histogram of the obstacle labels under them;
//   contacts:    the support cells of one offset, in run order.
// Only the bottom of a run can meet an obstacle when the object falls (the point below any other point of a run is the object),
// so a run [z0, z1] needs one look-up per offset: b, the highest obstacle at or below its raised top.
#include <cub/cub.cuh>

#include <climits>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "ray_ops.cuh"
#include "sweep_grid.cuh"

namespace dmnerf {

namespace {

constexpr int TILE = 32;                      // column pass: 32 columns x 32 heights per step
constexpr int CP_WARPS = 8;
constexpr int RUN_WARPS = 8;                  // runs: one warp per column
constexpr int MAP_WARPS = 8;                  // map: one warp per offset
constexpr int CT_THREADS = 256;               // contacts: one block
constexpr int MV_THREADS = 256;               // moved object: one thread per (column, height)
constexpr int N_BINS = DMNERF_MAX_INS + 1;
constexpr unsigned FULL = 0xffffffffu;

// The placement's axes: linear index strides of h1, h2 and the down axis, and whether the height runs against the index.
struct Frame {
  int64_t s1, s2, sa;
  int dim;
  int flip;                                   // 1: y = dim - 1 - idx_axis (down is +e_axis)
  int height_fast;                            // the down axis is the grid's fastest index
};

__device__ __forceinline__ int64_t point_of(const Frame& f, int h1, int h2, int y) {
  return h1 * f.s1 + h2 * f.s2 + (int64_t)(f.flip ? f.dim - 1 - y : y) * f.sa;
}

// What the placed object and the obstacles are (DESIGN.md, "Object placement", "Moving objects together"): S = label in the
// group, solid, kept by the piece for that label; O = solid, label among the obstacles, not vacated (label in the group and in the
// piece -- every point without one -- or rest_drop).  A COPY (DESIGN.md, "Copying objects") vacates nothing: its own labels' solid
// points are obstacles like any other.
struct Placed {
  Region piece;                               // bits NULL: the whole labels
  ObjMask obstacles;
  ObjMask group;                              // the labels placed together ({label} for one object)
  int label, rest_drop;
};

// The status a call reads back: the grid check's flags, the object's box, height range and sums (over its points, of h1, h2
// and y), its points and its runs.  Integer atomics only, so every field is independent of their order.
struct Status {
  int bad;
  int box[6];                                 // h1 lo, hi, h2 lo, hi, y lo, hi
  int n_cells;                                // contacts pass: support runs written; drop at the offset (-1: blocked)
  int drop;
  int pad;
  unsigned long long points, runs, sum[3];
};

struct __align__(8) ObjRun {
  int16_t h1, h2, z0, z1;
};

template <bool COPY>
__device__ __forceinline__ void classify(const Frame& f, const GridXform& g, const Placed& m, const float* __restrict__ occ,
                                         const int16_t* __restrict__ labels, float level, int64_t p, bool& obst, bool& obj) {
  const float v = occ[p];
  const int l = labels[p];
  const bool solid = v > level && l >= 0 && l <= DMNERF_MAX_INS;
  obst = solid && obj_kept(m.obstacles, l);
  obj = false;
  if (solid && in_group(m.group, l)) {
    bool keep = true;
    if (m.piece.bits != nullptr) {
      float q[3];
      sweep_point(g, p, q);
      keep = !region_drops(m.piece, l, q[0], q[1], q[2]);
    }
    obj = keep;
    if (!COPY && (keep || m.rest_drop)) obst = false;            // vacated by the move
  }
}

// A block takes 32 consecutive columns and walks their heights 32 at a time.  The load reads the grid along its fastest index
// (the height when the down axis is the fastest, the column's h2 otherwise); each warp then scans 4 of the columns with its lanes
// on the heights (a warp max-scan, carried from chunk to chunk) and writes 32 contiguous table entries and, with OBJECT (the
// object as it lies), object bytes.  A moved object's bytes come from place_moved_kernel; the table never depends on the move.
// COPY: the table of a copy's scene, whose own label stays (always with a base, so never with OBJECT).
template <bool OBJECT, bool COPY = false>
__global__ void __launch_bounds__(CP_WARPS * 32) place_column_kernel(const Frame f, const GridXform g, const Placed m,
                                                                     const float* __restrict__ occ, const int16_t* __restrict__ labels,
                                                                     float level, int16_t* __restrict__ table,
                                                                     uint8_t* __restrict__ object) {
  __shared__ uint8_t s[TILE][TILE + 1];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t n_cols = (int64_t)f.dim * f.dim;
  const int64_t c0 = (int64_t)blockIdx.x * TILE;
  int carry[TILE / CP_WARPS];
#pragma unroll
  for (int k = 0; k < TILE / CP_WARPS; ++k) carry[k] = -1;
  for (int y0 = 0; y0 < f.dim; y0 += TILE) {
    for (int r = w; r < TILE; r += CP_WARPS) {
      const int cl = f.height_fast ? r : lane, yl = f.height_fast ? lane : r;
      const int64_t c = c0 + cl;
      const int y = y0 + yl;
      uint8_t bits = 0;
      if (c < n_cols && y < f.dim) {
        bool obst, obj;
        classify<COPY>(f, g, m, occ, labels, level, point_of(f, (int)(c / f.dim), (int)(c % f.dim), y), obst, obj);
        bits = (obst ? 1 : 0) | (obj ? 2 : 0);
      }
      s[cl][yl] = bits;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < TILE / CP_WARPS; ++k) {
      const int cl = w + k * CP_WARPS;
      const int64_t c = c0 + cl;
      const int y = y0 + lane;
      const int bits = s[cl][lane];
      int v = (bits & 1) ? y : -1;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int o = __shfl_up_sync(FULL, v, d);
        if (lane >= d) v = max(v, o);
      }
      v = max(v, carry[k]);
      carry[k] = __shfl_sync(FULL, v, 31);
      if (c < n_cols && y < f.dim) {
        table[c * f.dim + y] = (int16_t)v;
        if (OBJECT) object[c * f.dim + y] = (uint8_t)(bits >> 1);
      }
    }
    __syncthreads();
  }
}

// The object as the move e leaves it (DESIGN.md, "Turned placements"), one thread per (column, height) in the object bytes
// order: point p belongs to it when src(p) of the collision checks holds -- q = edit_target(e, p) in the box B, labels[q] in the
// move's group, occ[q] > level and the piece keeps the target t for that label.  Points the move carries outside the grid are lost, as in the edited sweep.
__global__ void __launch_bounds__(MV_THREADS) place_moved_kernel(const Frame f, const GridXform g, const EditMove e,
                                                                 const float* __restrict__ occ, const int16_t* __restrict__ labels,
                                                                 float level, uint8_t* __restrict__ object) {
  const int64_t o = (int64_t)blockIdx.x * MV_THREADS + threadIdx.x, d = f.dim;
  if (o >= d * d * d) return;
  const int64_t c = o / d;
  float p[3], t[3];
  double q[3];
  sweep_point(g, point_of(f, (int)(c / d), (int)(c % d), (int)(o % d)), p);
  bool src = edit_target(e.trans, e.inv, e.b, e.lo, e.hi, !e.empty, p, t, q);
  if (src) {
    const int64_t qi = ((int64_t)q[0] * d + (int64_t)q[1]) * d + (int64_t)q[2];
    const int lq = labels[qi];
    src = in_group(e.group, lq) && occ[qi] > level && (e.piece.bits == nullptr || !region_drops(e.piece, lq, t[0], t[1], t[2]));
  }
  object[o] = src ? 1 : 0;
}

// One warp per column: its runs (a bottom: object here, not below; a top: object here, not above) and its points, with the
// object's box, height range and sums accumulated once per column.
__global__ void __launch_bounds__(RUN_WARPS * 32) place_run_count_kernel(int dim, const uint8_t* __restrict__ object,
                                                                         int32_t* __restrict__ counts, Status* __restrict__ st) {
  const int lane = threadIdx.x & 31;
  const int64_t c = (int64_t)blockIdx.x * RUN_WARPS + (threadIdx.x >> 5);
  if (c >= (int64_t)dim * dim) return;
  const uint8_t* col = object + c * dim;
  int runs = 0, points = 0, ylo = INT_MAX, yhi = -1;
  unsigned long long ysum = 0;
  for (int y0 = 0; y0 < dim; y0 += 32) {
    const int y = y0 + lane;
    const bool here = y < dim && col[y];
    const bool below = here && y > 0 && col[y - 1];
    runs += __popc(__ballot_sync(FULL, here && !below));
    points += __popc(__ballot_sync(FULL, here));
    if (here) {
      ylo = min(ylo, y);
      yhi = max(yhi, y);
      ysum += (unsigned long long)y;
    }
  }
  ysum = __reduce_add_sync(FULL, (unsigned)ysum);                // < 2^32: at most 1024 heights of at most 1023
  ylo = __reduce_min_sync(FULL, ylo);
  yhi = __reduce_max_sync(FULL, yhi);
  if (lane == 0) {
    counts[c] = runs;
    if (points) {
      const int h1 = (int)(c / dim), h2 = (int)(c % dim);
      atomicMin(&st->box[0], h1);
      atomicMax(&st->box[1], h1);
      atomicMin(&st->box[2], h2);
      atomicMax(&st->box[3], h2);
      atomicMin(&st->box[4], ylo);
      atomicMax(&st->box[5], yhi);
      atomicAdd(&st->points, (unsigned long long)points);
      atomicAdd(&st->runs, (unsigned long long)runs);
      atomicAdd(&st->sum[0], (unsigned long long)h1 * points);
      atomicAdd(&st->sum[1], (unsigned long long)h2 * points);
      atomicAdd(&st->sum[2], ysum);
    }
  }
}

// One warp per column: the column's runs at offsets[c] .. offsets[c] + counts[c] - 1, bottom to top.  The k-th bottom and the
// k-th top of a column belong to its k-th run.
__global__ void __launch_bounds__(RUN_WARPS * 32) place_run_write_kernel(int dim, const uint8_t* __restrict__ object,
                                                                         const int32_t* __restrict__ counts,
                                                                         const int32_t* __restrict__ offsets, ObjRun* __restrict__ runs) {
  const int lane = threadIdx.x & 31;
  const int64_t c = (int64_t)blockIdx.x * RUN_WARPS + (threadIdx.x >> 5);
  if (c >= (int64_t)dim * dim || counts[c] == 0) return;
  const uint8_t* col = object + c * dim;
  ObjRun* out = runs + offsets[c];
  const unsigned below_me = (1u << lane) - 1u;
  int n_bot = 0, n_top = 0;
  for (int y0 = 0; y0 < dim; y0 += 32) {
    const int y = y0 + lane;
    const bool here = y < dim && col[y];
    const bool bot = here && !(y > 0 && col[y - 1]);
    const bool top = here && !(y + 1 < dim && col[y + 1]);
    const unsigned bm = __ballot_sync(FULL, bot), tm = __ballot_sync(FULL, top);
    if (bot) {
      ObjRun& r = out[n_bot + __popc(bm & below_me)];
      r.h1 = (int16_t)(c / dim);
      r.h2 = (int16_t)(c % dim);
      r.z0 = (int16_t)y;
    }
    if (top) out[n_top + __popc(tm & below_me)].z1 = (int16_t)y;
    n_bot += __popc(bm);
    n_top += __popc(tm);
  }
}

// b of run q at offset (u, v): the highest obstacle height at or below its raised top, -1 for none
__device__ __forceinline__ int obstacle_below(const Frame& f, const int16_t* __restrict__ table, const ObjRun& q, int u, int v,
                                              int lift) {
  return table[((int64_t)(q.h1 + u) * f.dim + (q.h2 + v)) * f.dim + (q.z1 + lift)];
}

__global__ void __launch_bounds__(MAP_WARPS * 32) place_map_kernel(const Frame f, const int16_t* __restrict__ table,
                                                                   const int16_t* __restrict__ labels, const ObjRun* __restrict__ runs,
                                                                   int64_t n_runs, int u_lo, int v_lo, int U, int V, int lift,
                                                                   int32_t* __restrict__ drop, int32_t* __restrict__ contacts,
                                                                   int16_t* __restrict__ support) {
  __shared__ uint32_t hist[MAP_WARPS][N_BINS];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t o = (int64_t)blockIdx.x * MAP_WARPS + w;
  if (o >= (int64_t)U * V) return;                               // warp-uniform; nothing below synchronises the block
  const int u = u_lo + (int)(o / V), v = v_lo + (int)(o % V);
  int fall = INT_MAX;
  bool blocked = false;
  for (int64_t r = lane; r < n_runs; r += 32) {
    const ObjRun q = runs[r];
    const int b = obstacle_below(f, table, q, u, v, lift), bot = q.z0 + lift;
    blocked |= b >= bot;
    fall = min(fall, bot - b - 1);                               // b = -1: down to height 0
  }
  if (__any_sync(FULL, blocked)) {
    if (lane == 0) {
      drop[o] = -1;
      contacts[o] = 0;
      support[o] = -1;
    }
    return;
  }
  fall = __reduce_min_sync(FULL, fall);
  for (int k = lane; k < N_BINS; k += 32) hist[w][k] = 0;
  __syncwarp();
  int n = 0;
  for (int64_t r = lane; r < n_runs; r += 32) {
    const ObjRun q = runs[r];
    const int b = obstacle_below(f, table, q, u, v, lift);
    if (b >= 0 && b == q.z0 + lift - fall - 1) {                 // the run's bottom rests on an obstacle point
      ++n;
      atomicAdd(&hist[w][labels[point_of(f, q.h1 + u, q.h2 + v, b)]], 1u);
    }
  }
  n = __reduce_add_sync(FULL, (unsigned)n);
  __syncwarp();
  unsigned best = 0;                                             // (runs << 8) | (127 - label): most runs, then lowest label
  for (int k = lane; k < N_BINS; k += 32) {
    const unsigned key = (hist[w][k] << 8) | (unsigned)(N_BINS - 1 - k);
    if (hist[w][k] && key > best) best = key;
  }
  best = __reduce_max_sync(FULL, best);
  if (lane == 0) {
    drop[o] = fall;
    contacts[o] = n;
    support[o] = n ? (int16_t)(N_BINS - 1 - (int)(best & 0xff)) : (int16_t)-1;
  }
}

// One block: the drop at (u, v) as the map computes it, then (h1 + u, h2 + v, label below) of every run resting on an obstacle,
// in run order (a block scan per 256 runs).
__global__ void __launch_bounds__(CT_THREADS) place_contacts_kernel(const Frame f, const int16_t* __restrict__ table,
                                                                    const int16_t* __restrict__ labels, const ObjRun* __restrict__ runs,
                                                                    int64_t n_runs, int u, int v, int lift, Status* __restrict__ st,
                                                                    int32_t* __restrict__ cells) {
  typedef cub::BlockScan<int, CT_THREADS> Scan;
  __shared__ typename Scan::TempStorage scan;
  __shared__ int s_fall[CT_THREADS / 32], s_blocked[CT_THREADS / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int fall = INT_MAX, blocked = 0;
  for (int64_t r = threadIdx.x; r < n_runs; r += CT_THREADS) {
    const ObjRun q = runs[r];
    const int b = obstacle_below(f, table, q, u, v, lift), bot = q.z0 + lift;
    blocked |= b >= bot;
    fall = min(fall, bot - b - 1);
  }
  fall = __reduce_min_sync(FULL, fall);
  blocked = __reduce_or_sync(FULL, (unsigned)blocked);
  if (lane == 0) {
    s_fall[w] = fall;
    s_blocked[w] = blocked;
  }
  __syncthreads();
  fall = INT_MAX;
  blocked = 0;
  for (int k = 0; k < CT_THREADS / 32; ++k) {
    fall = min(fall, s_fall[k]);
    blocked |= s_blocked[k];
  }
  if (blocked) {
    if (threadIdx.x == 0) {
      st->drop = -1;
      st->n_cells = 0;
    }
    return;                                                      // block-uniform
  }
  int written = 0;
  for (int64_t r0 = 0; r0 < n_runs; r0 += CT_THREADS) {
    const int64_t r = r0 + threadIdx.x;
    int flag = 0, b = -1;
    ObjRun q{};
    if (r < n_runs) {
      q = runs[r];
      b = obstacle_below(f, table, q, u, v, lift);
      flag = b >= 0 && b == q.z0 + lift - fall - 1;
    }
    int pos, total;
    Scan(scan).ExclusiveSum(flag, pos, total);
    if (flag) {
      int32_t* cell = cells + 3 * (int64_t)(written + pos);
      cell[0] = q.h1 + u;
      cell[1] = q.h2 + v;
      cell[2] = labels[point_of(f, q.h1 + u, q.h2 + v, b)];
    }
    written += total;
    __syncthreads();                                             // the scan's storage is reused
  }
  if (threadIdx.x == 0) {
    st->drop = fall;
    st->n_cells = written;
  }
}

// The checked grids and placement of a call, its buffers, and after object_runs the object's status, runs and offset range.
// occ / labels: the scene, which gives the obstacles, the vacated points and the labels under the object (the column pass, the
// map and the contacts); src_occ / src_labels: the grid a moved object is sampled from (place_moved_kernel).  They are the same
// grid except in a placement in an edited scene (DESIGN.md, "Arranging objects").
struct Prepared {
  Frame f;
  GridXform g;
  Placed m;
  bool copy;                                  // the object is a copy: the scene's points of its label stay obstacles
  const float* occ;
  const int16_t* labels;
  const float* src_occ;
  const int16_t* src_labels;
  float level;
  int lift;
  Status st;
  int16_t* table;
  uint8_t* object;
  int32_t *counts, *offsets;
  ObjRun* runs;
  Status* st_dev;
  int u_lo, v_lo, U, V;
};

enum { PLACED = 0, NO_POINTS = 1, TOP_OUT = 2 };   // dmnerf_placement_maps' status per base

// The host checks of every placement call, before any launch: the object's grid occ / labels and the scene.
int check(const float* occ, const int16_t* labels, const float* scene_occ, const int16_t* scene_labels, int dim, float level,
          const double* T16, const double* ext3, const dmnerf_placement* p, int copy, const uint32_t* group4, const char* who,
          Prepared& q) {
  DMN_CHECK(occ && labels && scene_occ && scene_labels && T16 && ext3 && p, "%s: NULL argument", who);
  DMN_CHECK(dim >= 2 && dim <= PLACE_MAX_DIM, "%s: dim %d out of range [2, %d]", who, dim, PLACE_MAX_DIM);
  if (sweep_grid_check(T16, ext3, dim, level, who)) return 1;
  DMN_CHECK(p->label >= 0 && p->label <= DMNERF_MAX_INS, "%s: label %d outside [0, %d]", who, p->label, DMNERF_MAX_INS);
  DMN_CHECK(p->axis >= 0 && p->axis <= 2, "%s: down axis %d is not 0, 1 or 2", who, p->axis);
  DMN_CHECK(p->sign == 1 || p->sign == -1, "%s: the sign of down along its axis must be +1 or -1, got %d", who, p->sign);
  DMN_CHECK(p->lift >= 0 && p->lift <= dim - 1, "%s: lift %d takes the object out of the grid [0, %d]", who, p->lift, dim - 1);
  DMN_CHECK(copy == 0 || copy == 1, "%s: copy flag %d is not 0 or 1", who, copy);
  DMN_CHECK(!copy || !p->rest_drop, "%s: a copy cannot drop the rest of its label (it vacates nothing)", who);
  q.copy = copy != 0;
  Placed& m = q.m;
  if (label_group(p->label, group4, DMNERF_MAX_INS, m.group, who, -1)) return 1;
  if (piece_region(p->piece, p->label, m.piece, who, 0)) return 1;
  for (int k = 0; k < 4; ++k) m.obstacles.w[k] = p->obstacles[k];
  m.label = p->label;
  m.rest_drop = p->rest_drop ? 1 : 0;
  const int64_t d = dim, stride[3] = {d * d, d, 1};
  const int h1 = p->axis == 0 ? 1 : 0, h2 = p->axis == 2 ? 1 : 2;
  Frame& f = q.f;
  f.s1 = stride[h1];
  f.s2 = stride[h2];
  f.sa = stride[p->axis];
  f.dim = dim;
  f.flip = p->sign == 1 ? 1 : 0;
  f.height_fast = p->axis == 2 ? 1 : 0;
  q.g = make_xform(T16, ext3, dim);
  q.occ = scene_occ;
  q.labels = scene_labels;
  q.src_occ = occ;
  q.src_labels = labels;
  q.level = level;
  q.lift = p->lift;
  return 0;
}

// base (row-major 3x4) and the source box B of a moved placement as the edit move the shared checks take: finite, det > 0, B
// inside the grid and not inverted (the empty box: no point), the piece applying to the label; the group checked by check().
int base_move(const dmnerf_placement* p, const ObjMask& group, const double* base12, const int32_t* box6, const double* T16,
              const double* ext3, int dim, EditMove& e, const char* who, int i) {
  dmnerf_edit_move d;
  memset(&d, 0, sizeof(d));
  d.label = p->label;
  d.rest_drop = p->rest_drop;
  memcpy(d.trans, base12, sizeof(d.trans));
  memcpy(d.box, box6, sizeof(d.box));
  d.piece = p->piece;
  return edit_move_from_abi(d, T16, ext3, dim, DMNERF_MAX_INS, e, who, i, group.w);
}

// The buffers, the grid check (of both grids when the scene is not the object's grid) and the column pass: the column table,
// and the bytes of the unmoved object when `unmoved`.
int columns(PlaceState& s, Prepared& q, bool unmoved, cudaStream_t stream) {
  const int64_t d = q.f.dim, n = d * d * d, n_cols = d * d;
  if (s.table.get((size_t)n, &q.table) || s.object.get((size_t)n, &q.object) || s.counts.get((size_t)n_cols, &q.counts) ||
      s.offsets.get((size_t)n_cols, &q.offsets) || s.status.get(1, &q.st_dev))
    return 2;
  Status init{};
  for (int a = 0; a < 3; ++a) {
    init.box[2 * a] = INT_MAX;
    init.box[2 * a + 1] = -1;
  }
  DMN_CUDA(cudaMemcpyAsync(q.st_dev, &init, sizeof(init), cudaMemcpyHostToDevice, stream));
  if (launch_grid_check(q.occ, q.labels, n, DMNERF_MAX_INS + 1, &q.st_dev->bad, stream)) return 2;
  if ((q.src_occ != q.occ || q.src_labels != q.labels) &&
      launch_grid_check(q.src_occ, q.src_labels, n, DMNERF_MAX_INS + 1, &q.st_dev->bad, stream))
    return 2;
  const unsigned blocks = (unsigned)((n_cols + TILE - 1) / TILE);
  if (unmoved)
    place_column_kernel<true><<<blocks, CP_WARPS * 32, 0, stream>>>(q.f, q.g, q.m, q.occ, q.labels, q.level, q.table, q.object);
  else if (q.copy)
    place_column_kernel<false, true><<<blocks, CP_WARPS * 32, 0, stream>>>(q.f, q.g, q.m, q.occ, q.labels, q.level, q.table, nullptr);
  else
    place_column_kernel<false><<<blocks, CP_WARPS * 32, 0, stream>>>(q.f, q.g, q.m, q.occ, q.labels, q.level, q.table, nullptr);
  DMN_LAUNCH_OK();
  return 0;
}

// The object's bytes when it is moved by `base` (NULL: as the column pass wrote them), its runs and the status read-back, after
// which *why says whether it can be placed (PLACED) or why not.  The grid check's flags fail the call.
int object_runs(PlaceState& s, Prepared& q, const EditMove* base, bool first, const char* who, int* why, cudaStream_t stream) {
  const int64_t d = q.f.dim, n = d * d * d, n_cols = d * d;
  if (!first) {                                                  // the grid check's flags were read with the first base
    Status init{};
    for (int a = 0; a < 3; ++a) {
      init.box[2 * a] = INT_MAX;
      init.box[2 * a + 1] = -1;
    }
    DMN_CUDA(cudaMemcpyAsync(q.st_dev, &init, sizeof(init), cudaMemcpyHostToDevice, stream));
  }
  if (base) {
    place_moved_kernel<<<(unsigned)((n + MV_THREADS - 1) / MV_THREADS), MV_THREADS, 0, stream>>>(q.f, q.g, *base, q.src_occ,
                                                                                                 q.src_labels, q.level, q.object);
    DMN_LAUNCH_OK();
  }
  const unsigned col_blocks = (unsigned)((n_cols + RUN_WARPS - 1) / RUN_WARPS);
  place_run_count_kernel<<<col_blocks, RUN_WARPS * 32, 0, stream>>>(q.f.dim, q.object, q.counts, q.st_dev);
  DMN_LAUNCH_OK();
  size_t tmp_bytes = 0;
  DMN_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, q.counts, q.offsets, (int)n_cols, stream));
  char* tmp;
  if (s.temp.get(tmp_bytes, &tmp)) return 2;
  DMN_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, q.counts, q.offsets, (int)n_cols, stream));
  if (const int rc = read_checked(q.st_dev, &q.st, sizeof(Status), DMNERF_MAX_INS, who, stream)) return rc;
  const Status& st = q.st;
  *why = st.points == 0 ? NO_POINTS : (st.box[5] + q.lift > q.f.dim - 1 ? TOP_OUT : PLACED);
  if (*why != PLACED) return 0;
  if (s.runs.get((size_t)st.runs, &q.runs)) return 2;
  place_run_write_kernel<<<col_blocks, RUN_WARPS * 32, 0, stream>>>(q.f.dim, q.object, q.counts, q.offsets, q.runs);
  DMN_LAUNCH_OK();
  q.u_lo = -st.box[0];
  q.v_lo = -st.box[2];
  q.U = q.f.dim - (st.box[1] - st.box[0]);
  q.V = q.f.dim - (st.box[3] - st.box[2]);
  return 0;
}

// A placement that cannot be made fails a one-object call with its reason.
int unplaced(const Prepared& q, int why, bool moved, const char* who) {
  DMN_CHECK(why != NO_POINTS, "%s: label %d has no solid points%s", who, q.m.label,
            moved ? " after the move" : (q.m.piece.bits ? " in its piece" : ""));
  DMN_CHECK(why != TOP_OUT, "%s: lift %d takes the object's top (height %d) out of the grid [0, %d]", who, q.lift, q.st.box[5],
            q.f.dim - 1);
  return 0;
}

int launch_map(const Prepared& q, int32_t* drop, int32_t* contacts, int16_t* support, cudaStream_t st) {
  const int64_t offsets = (int64_t)q.U * q.V;
  place_map_kernel<<<(unsigned)((offsets + MAP_WARPS - 1) / MAP_WARPS), MAP_WARPS * 32, 0, st>>>(
      q.f, q.table, q.labels, q.runs, (int64_t)q.st.runs, q.u_lo, q.v_lo, q.U, q.V, q.lift, drop, contacts, support);
  DMN_LAUNCH_OK();
  return 0;
}

void fill_info(const Prepared& q, dmnerf_placement_info* info) {
  memset(info, 0, sizeof(*info));
  info->offset_lo[0] = q.u_lo;
  info->offset_lo[1] = q.v_lo;
  info->offsets[0] = q.U;
  info->offsets[1] = q.V;
  info->height[0] = q.st.box[4];
  info->height[1] = q.st.box[5];
  info->runs = (int64_t)q.st.runs;
  info->points = (int64_t)q.st.points;
  for (int a = 0; a < 3; ++a) info->sum[a] = (int64_t)q.st.sum[a];
}

// The support cells of offset (u, v) of a prepared object, read back to the host.
int contacts_at(PlaceState& s, const Prepared& q, int u, int v, int32_t* cells_host, int64_t max_cells, int64_t* n_cells_host,
                int32_t* drop_host, const char* who, cudaStream_t st) {
  DMN_CHECK(u >= q.u_lo && u < q.u_lo + q.U && v >= q.v_lo && v < q.v_lo + q.V,
            "%s: offset (%d, %d) outside the offsets [%d, %d] x [%d, %d] that keep the object inside the grid", who, u, v, q.u_lo,
            q.u_lo + q.U - 1, q.v_lo, q.v_lo + q.V - 1);
  int32_t* cells;
  if (s.cells.get((size_t)3 * q.st.runs, &cells)) return 2;
  place_contacts_kernel<<<1, CT_THREADS, 0, st>>>(q.f, q.table, q.labels, q.runs, (int64_t)q.st.runs, u, v, q.lift, q.st_dev, cells);
  DMN_LAUNCH_OK();
  Status h;
  DMN_CUDA(cudaMemcpyAsync(&h, q.st_dev, sizeof(h), cudaMemcpyDeviceToHost, st));
  DMN_CUDA(cudaStreamSynchronize(st));
  DMN_CHECK(h.n_cells <= max_cells, "%s: %d support runs need room for as many cells, got %lld", who, h.n_cells, (long long)max_cells);
  if (h.n_cells) {
    DMN_CUDA(cudaMemcpyAsync(cells_host, cells, (size_t)h.n_cells * 3 * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    DMN_CUDA(cudaStreamSynchronize(st));
  }
  *n_cells_host = h.n_cells;
  *drop_host = h.drop;
  return 0;
}

}  // namespace

int placement_map(PlaceState& s, const float* occ, const int16_t* labels, int dim, float level, const double* T16, const double* ext3,
                  const dmnerf_placement* p, int32_t* drop, int32_t* contacts, int16_t* support, dmnerf_placement_info* info,
                  cudaStream_t st) {
  const char* who = "placement_map";
  DMN_CHECK(drop && contacts && support && info, "%s: NULL argument", who);
  memset(info, 0, sizeof(*info));
  Prepared q;
  int why;
  if (check(occ, labels, occ, labels, dim, level, T16, ext3, p, 0, nullptr, who, q)) return 1;
  if (const int rc = columns(s, q, true, st)) return rc;
  if (const int rc = object_runs(s, q, nullptr, true, who, &why, st)) return rc;
  if (unplaced(q, why, false, who)) return 1;
  if (const int rc = launch_map(q, drop, contacts, support, st)) return rc;
  fill_info(q, info);
  return 0;
}

int placement_maps(PlaceState& s, const float* occ, const int16_t* labels, const float* scene_occ, const int16_t* scene_labels, int dim,
                   float level, const double* T16, const double* ext3, const dmnerf_placement* p, int copy, const uint32_t* group_host,
                   const double* bases_host, const int32_t* box_host, int n_bases, int32_t* drop, int32_t* contacts, int16_t* support, dmnerf_placement_info* info,
                   int32_t* status, cudaStream_t st, const char* who) {
  if (!who) who = occ == scene_occ && labels == scene_labels ? "placement_maps" : "placement_maps_in_scene";
  DMN_CHECK(drop && contacts && support && info && status, "%s: NULL argument", who);
  DMN_CHECK(n_bases >= 1 && n_bases <= DMNERF_MAX_BASES, "%s: between 1 and %d bases are supported, got %d", who, DMNERF_MAX_BASES,
            n_bases);
  DMN_CHECK(bases_host && box_host, "%s: bases or box is NULL", who);
  for (int i = 0; i < n_bases; ++i) {
    memset(info + i, 0, sizeof(*info));
    status[i] = NO_POINTS;
  }
  Prepared q;
  if (check(occ, labels, scene_occ, scene_labels, dim, level, T16, ext3, p, copy, group_host, who, q)) return 1;
  std::vector<EditMove> e(n_bases);
  for (int i = 0; i < n_bases; ++i)
    if (base_move(p, q.m.group, bases_host + 12 * i, box_host, T16, ext3, dim, e[i], who, i)) return 1;
  if (const int rc = columns(s, q, false, st)) return rc;
  const int64_t plane = (int64_t)dim * dim;
  for (int i = 0; i < n_bases; ++i) {
    int why;
    if (const int rc = object_runs(s, q, &e[i], i == 0, who, &why, st)) return rc;
    status[i] = why;
    if (why != PLACED) continue;
    if (const int rc = launch_map(q, drop + i * plane, contacts + i * plane, support + i * plane, st)) return rc;
    fill_info(q, info + i);
  }
  return 0;
}

int placement_contacts(PlaceState& s, const float* occ, const int16_t* labels, const float* scene_occ, const int16_t* scene_labels,
                       int dim, float level, const double* T16, const double* ext3, const dmnerf_placement* p, int copy,
                       const uint32_t* group_host, const double* base_host, const int32_t* box_host, int u, int v, int32_t* cells_host, int64_t max_cells, int64_t* n_cells_host,
                       int32_t* drop_host, cudaStream_t st, const char* who) {
  const bool moved = base_host != nullptr;
  if (!who)
    who = !moved ? "placement_contacts"
                 : (occ == scene_occ && labels == scene_labels ? "placement_contacts_moved" : "placement_contacts_in_scene");
  DMN_CHECK(n_cells_host && drop_host && max_cells >= 0 && (max_cells == 0 || cells_host), "%s: bad output arguments", who);
  *n_cells_host = 0;
  *drop_host = -1;
  Prepared q;
  EditMove e;
  int why;
  DMN_CHECK(moved || !copy, "%s: a copy is placed through a base", who);
  if (check(occ, labels, scene_occ, scene_labels, dim, level, T16, ext3, p, copy, group_host, who, q)) return 1;
  if (moved) {
    DMN_CHECK(box_host, "%s: box is NULL", who);
    if (base_move(p, q.m.group, base_host, box_host, T16, ext3, dim, e, who, 0)) return 1;
  }
  if (const int rc = columns(s, q, !moved, st)) return rc;
  if (const int rc = object_runs(s, q, moved ? &e : nullptr, true, who, &why, st)) return rc;
  if (unplaced(q, why, moved, who)) return 1;
  return contacts_at(s, q, u, v, cells_host, max_cells, n_cells_host, drop_host, who, st);
}

}  // namespace dmnerf
