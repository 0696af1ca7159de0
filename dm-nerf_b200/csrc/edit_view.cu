// Tracing the hits of an edited grid to the moves that placed them (DESIGN.md, "Viewing the labelled grid", "Colouring an edited
// view"): per cast ray with a hit voxel q, the grid-only edit (collide.cu grid_edit_kernel) replayed at q's sweep point alone,
// from the source grid's (occ, label) at q, with the same edit_rule, targets, box, piece, copy and group decisions.  The last
// move that took at q is the hit's provenance m*; the colour point is the hit point o + depth d pulled back through m* (its
// target, as the moved render takes it) and the colour direction is the moved render's direction before its normalisation.  The
// replay's (occ, label) must equal the viewed grid's at q bit for bit; a hit where it does not is counted, so a grid that is not
// the grid-only edit of that source by those moves is reported rather than coloured wrongly.
#include <cmath>
#include <cstring>

#include "common.cuh"
#include "ray_ops.cuh"
#include "sweep_grid.cuh"

namespace dmnerf {

namespace {

constexpr int EV_THREADS = 128;
constexpr unsigned FULL = 0xffffffffu;

// The checked moves of one call, in order, with their deformations (n_knots 0: rigid) and copy flags.
struct EditView {
  EditMove m[DMNERF_MAX_MOVES];
  Deform df[DMNERF_MAX_MOVES];
  int32_t copy[DMNERF_MAX_MOVES];
  GridXform g;
  float level;
  int32_t n_moves;
};

// One thread per ray r.  counts [2]: the hits whose replay differs from the viewed grid (and the rays whose voxel index is
// outside [-1, dim^3)), then the bad indices alone.  move_out [n] = m* (-1: no hit or no take), point_out [n][3] = the colour
// point (NaN: no hit), dir_out [n][3] = the colour direction, not normalised (0: no hit).
__global__ void __launch_bounds__(EV_THREADS) edit_source_kernel(const EditView v, const float* __restrict__ occ,
                                                                 const int16_t* __restrict__ labels, const float* __restrict__ src_occ,
                                                                 const int16_t* __restrict__ src_labels,
                                                                 const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                                                 const float* __restrict__ t_in, const int32_t* __restrict__ voxel_in,
                                                                 int64_t n, int32_t* __restrict__ move_out, float* __restrict__ point_out,
                                                                 float* __restrict__ dir_out, unsigned long long* __restrict__ counts) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool mismatch = false, bad = false;
  if (r < n) {
    const int64_t d = v.g.dim, q = voxel_in[r];
    int m_star = -1;
    float pt[3] = {NAN, NAN, NAN}, dir[3] = {0.0f, 0.0f, 0.0f};
    bad = q < -1 || q >= d * d * d;
    if (!bad && q >= 0) {
      float x[3];
      sweep_point(v.g, q, x);
      float o = src_occ[q];
      int l = src_labels[q];
      for (int k = 0; k < v.n_moves; ++k) {
        const EditMove& e = v.m[k];
        float t[3];
        double qt[3];
        bool in_box = !e.empty;
        if (v.df[k].n_knots)
          edit_target_deformed(e.trans, v.df[k], e.inv, e.b, e.lo, e.hi, in_box, x, t, qt);
        else
          in_box = edit_target(e.trans, e.inv, e.b, e.lo, e.hi, in_box, x, t, qt);
        auto target = [&](int& lt, float& ot) {
          const int64_t qi = ((int64_t)qt[0] * d + (int64_t)qt[1]) * d + (int64_t)qt[2];
          lt = src_labels[qi];
          ot = src_occ[qi];
        };
        auto drops = [&](int lt) { return region_drops(e.piece, lt, t[0], t[1], t[2]); };
        auto in_piece = [&](bool& b, int lp) { b = e.piece.bits == nullptr || !region_drops(e.piece, lp, x[0], x[1], x[2]); };
        auto take = [&](float ot, int lt) {
          o = ot;
          l = lt;
          m_star = k;
        };
        auto vacate = [&] { o = 0.0f; };
        if (v.copy[k])
          edit_rule<true>(e, in_box, target, o, l, v.level, drops, in_piece, take, vacate);
        else
          edit_rule<false>(e, in_box, target, o, l, v.level, drops, in_piece, take, vacate);
      }
      mismatch = __float_as_uint(o) != __float_as_uint(occ[q]) || l != (int)labels[q];
      // the hit point as cast_grid returns it: o + depth d, multiply then add, each rounded once
      const float ro[3] = {rays_o[3 * r], rays_o[3 * r + 1], rays_o[3 * r + 2]};
      const float rd[3] = {rays_d[3 * r], rays_d[3 * r + 1], rays_d[3 * r + 2]};
      const float depth = t_in[r];
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        pt[a] = __fadd_rn(ro[a], __fmul_rn(depth, rd[a]));
        dir[a] = rd[a];
      }
      if (m_star >= 0) {
        // the target of the hit point under m* and the moved render's direction there (move_target_kernel, not normalised)
        const EditMove& e = v.m[m_star];
        const Deform& df = v.df[m_star];
        float t[3];
        double qt[3], w[3];
        bool in_box = true;
#pragma unroll
        for (int a = 0; a < 3; ++a) w[a] = moved_vector(e.trans, a, rd);
        if (df.n_knots) {
          const Pulled P = edit_target_deformed(e.trans, df, e.inv, e.b, e.lo, e.hi, in_box, pt, t, qt);
          double wp[3];
          deform_direction(df, P, w, wp);
#pragma unroll
          for (int a = 0; a < 3; ++a) dir[a] = __double2float_rn(wp[a]);
        } else {
          edit_target(e.trans, e.inv, e.b, e.lo, e.hi, in_box, pt, t, qt);
#pragma unroll
          for (int a = 0; a < 3; ++a) dir[a] = __double2float_rn(w[a]);
        }
#pragma unroll
        for (int a = 0; a < 3; ++a) pt[a] = t[a];
      }
    }
    move_out[r] = m_star;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      point_out[3 * r + a] = pt[a];
      dir_out[3 * r + a] = dir[a];
    }
  }
  const unsigned mis = __ballot_sync(FULL, mismatch || bad), nbad = __ballot_sync(FULL, bad);
  if ((threadIdx.x & 31) == 0) {
    if (mis) atomicAdd(counts, (unsigned long long)__popc(mis));
    if (nbad) atomicAdd(counts + 1, (unsigned long long)__popc(nbad));
  }
}

}  // namespace

int grid_edit_source(InventoryState& s, const float* occ, const int16_t* labels, const float* src_occ, const int16_t* src_labels,
                     const dmnerf_render_moves* moves, const int32_t* copies_host, const uint32_t* groups_host,
                     const dmnerf_deformation* deformations_host, const float* rays_o, const float* rays_d, const float* t_in,
                     const int32_t* voxel_in, int64_t n, int32_t* move_out, float* point_out, float* dir_out,
                     int64_t* mismatched_host, cudaStream_t st) {
  const char* who = "grid_edit_source";
  DMN_CHECK(moves != nullptr, "%s: moves is NULL", who);
  const int nm = moves->n_moves;
  if (deformations_check(deformations_host, nm > 0 && nm <= DMNERF_MAX_MOVES ? nm : 0, who)) return 1;
  DMN_CHECK(occ && labels && src_occ && src_labels && mismatched_host, "%s: NULL argument", who);
  DMN_CHECK(nm >= 1 && nm <= DMNERF_MAX_MOVES, "%s: between 1 and %d moves are supported, got %d", who, DMNERF_MAX_MOVES, nm);
  DMN_CHECK(moves->moves != nullptr, "%s: moves->moves is NULL", who);
  const int dim = moves->dim;
  if (sweep_grid_check(moves->transform, moves->extents, dim, moves->level, who)) return 1;
  DMN_CHECK(dim <= REGION_MAX_DIM, "%s: dim %d out of range [2, %d]", who, dim, REGION_MAX_DIM);
  DMN_CHECK(n >= 0, "%s: n %lld < 0", who, (long long)n);
  DMN_CHECK(n == 0 || (rays_o && rays_d && t_in && voxel_in && move_out && point_out && dir_out),
            "%s: a ray, cast or output pointer is NULL", who);
  // the viewed (edited) grid is checked against a replay from the source: they must be separate grids
  const int64_t npts = (int64_t)dim * dim * dim;
  auto apart = [](const void* a, size_t na, const void* b, size_t nb) {
    const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
    return x + na <= y || y + nb <= x;
  };
  const size_t fo = (size_t)npts * sizeof(float), lb = (size_t)npts * sizeof(int16_t);
  DMN_CHECK(apart(src_occ, fo, occ, fo) && apart(src_occ, fo, labels, lb) && apart(src_labels, lb, occ, fo) &&
                apart(src_labels, lb, labels, lb),
            "%s: the source and state grids overlap in memory (the state must be a separate copy)", who);
  EditView v;
  memset(&v, 0, sizeof(v));
  for (int i = 0; i < nm; ++i)
    if (edit_move_from_abi(moves->moves[i], moves->transform, moves->extents, dim, DMNERF_MAX_INS, v.m[i], who, i,
                           groups_host ? groups_host + 4 * i : nullptr))
      return 1;
  if (copy_flags_check(moves->moves, copies_host, groups_host, nm, true, who)) return 1;
  if (int rc = deformations_from_abi(deformations_host, nm, s.knots, v.df, nullptr, who, st)) return rc;
  for (int i = 0; i < nm; ++i) v.copy[i] = copies_host ? copies_host[i] : 0;
  v.g = make_xform(moves->transform, moves->extents, dim);
  v.level = moves->level;
  v.n_moves = nm;
  if (n == 0) {
    *mismatched_host = 0;
    return 0;
  }
  unsigned long long* counts;
  if (s.out.get(2, &counts)) return 2;
  DMN_CUDA(cudaMemsetAsync(counts, 0, 2 * sizeof(unsigned long long), st));
  edit_source_kernel<<<(unsigned)((n + EV_THREADS - 1) / EV_THREADS), EV_THREADS, 0, st>>>(
      v, occ, labels, src_occ, src_labels, rays_o, rays_d, t_in, voxel_in, n, move_out, point_out, dir_out, counts);
  DMN_LAUNCH_OK();
  unsigned long long h[2];
  DMN_CUDA(cudaMemcpyAsync(h, counts, sizeof(h), cudaMemcpyDeviceToHost, st));
  DMN_CUDA(cudaStreamSynchronize(st));
  DMN_CHECK(h[1] == 0, "%s: %llu cast voxel indices outside [-1, %lld)", who, h[1], (long long)npts);
  *mismatched_host = (int64_t)h[0];
  return 0;
}

}  // namespace dmnerf
