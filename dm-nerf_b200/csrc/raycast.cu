// Casting camera rays through a labelled grid (DESIGN.md, "Viewing the labelled grid"): per ray the first solid, kept voxel, its
// entry depth, label, linear index and a normal, with no network.  Grid point q owns the cube [q - 1/2, q + 1/2]^3; a ray is
// u(t) = u0 + t w in index space, u0 = inv (o - b) and w = inv d with the grid's index map (sweep_grid.cuh).  Every fp64 expression
// is rounded once per operation (the _rn intrinsics, no contraction) and every boundary time is computed directly from the voxel
// index, never accumulated, so that oracle/grid_cast_oracle.py visits the same voxels and returns the same bits.
//
// The walk is flat, one voxel per step.  A mask of empty 8^3 bricks, built per call and skipped in one step per brick, gave the
// same bits but measured slower on an H100 at grid_dim 256 and 512 (DESIGN.md, "Viewing the labelled grid"), so it is not used.
#include <cmath>
#include <cstring>

#include "common.cuh"
#include "sweep_grid.cuh"

namespace dmnerf {

namespace {

constexpr int CAST_THREADS = 128;

struct CastGrid {
  double inv[9], b[3];
  int dim;
  float level;
  ObjMask keep;
  int masked;                                // 0: every label kept
};

__device__ __forceinline__ bool kept_label(const CastGrid& g, int l) { return !g.masked || in_group(g.keep, l); }

__device__ __forceinline__ bool solid_at(const CastGrid& g, const float* __restrict__ occ, const int16_t* __restrict__ labels,
                                         int64_t p) {
  return __ldg(occ + p) > g.level && kept_label(g, __ldg(labels + p));
}

// The time u_a(t) reaches the boundary of voxel index q on the side the ray leaves it (s: +1 or -1 with w_a): (q + s/2 - u0) / w.
__device__ __forceinline__ double boundary(int q, int s, double u0, double w) {
  return __ddiv_rn(__dsub_rn((double)q + 0.5 * (double)s, u0), w);
}

// Whether axis b's boundary at time tb comes before axis a's at ta in the traversal's order (ties: the lower axis first).
__device__ __forceinline__ bool before(double tb, int b, double ta, int a) { return tb < ta || (tb == ta && b < a); }

// x[a] without dynamic indexing (a local array indexed at run time would live on the stack)
__device__ __forceinline__ double pick(int a, const double (&x)[3]) { return a == 0 ? x[0] : (a == 1 ? x[1] : x[2]); }

// n = -inv^T g (the index-space gradient g in the network frame, pointing out of the solid) -> |n|^2
__device__ __forceinline__ double normal_from(const double* inv, const double g[3], double n[3]) {
#pragma unroll
  for (int c = 0; c < 3; ++c)
    n[c] = -__dadd_rn(__dadd_rn(__dmul_rn(inv[c], g[0]), __dmul_rn(inv[3 + c], g[1])), __dmul_rn(inv[6 + c], g[2]));
  return __dadd_rn(__dadd_rn(__dmul_rn(n[0], n[0]), __dmul_rn(n[1], n[1])), __dmul_rn(n[2], n[2]));
}

__global__ void __launch_bounds__(CAST_THREADS) grid_cast_kernel(const float* __restrict__ occ, const int16_t* __restrict__ labels,
                                                                 CastGrid g,
                                                                 const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                                                 int64_t n, double near_t, double far_t, float* __restrict__ t_out,
                                                                 int16_t* __restrict__ label_out, int32_t* __restrict__ voxel_out,
                                                                 float* __restrict__ normal_out) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const float o[3] = {rays_o[3 * r], rays_o[3 * r + 1], rays_o[3 * r + 2]};
  const float d[3] = {rays_d[3 * r], rays_d[3 * r + 1], rays_d[3 * r + 2]};
  const int dim = g.dim;
  const double lo = -0.5, hi = (double)dim - 0.5;
  double u0[3], w[3];
  bool ok = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double* row = g.inv + 3 * a;
    const double dt[3] = {__dsub_rn((double)o[0], g.b[0]), __dsub_rn((double)o[1], g.b[1]), __dsub_rn((double)o[2], g.b[2])};
    u0[a] = __dadd_rn(__dadd_rn(__dmul_rn(row[0], dt[0]), __dmul_rn(row[1], dt[1])), __dmul_rn(row[2], dt[2]));
    w[a] = __dadd_rn(__dadd_rn(__dmul_rn(row[0], (double)d[0]), __dmul_rn(row[1], (double)d[1])), __dmul_rn(row[2], (double)d[2]));
    ok = ok && isfinite(u0[a]) && isfinite(w[a]);
  }
  ok = ok && (w[0] != 0.0 || w[1] != 0.0 || w[2] != 0.0);
  // the grid's cube [-1/2, dim - 1/2]^3: entry time (and its axis) and exit time
  double t_in = -INFINITY, t_out_grid = INFINITY;
  int in_axis = -1;
  int s[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    s[a] = w[a] > 0.0 ? 1 : -1;
    if (!ok) continue;
    if (w[a] == 0.0) {
      ok = u0[a] >= lo && u0[a] <= hi;
      continue;
    }
    const double ta = __ddiv_rn(__dsub_rn(s[a] > 0 ? lo : hi, u0[a]), w[a]);
    const double tb = __ddiv_rn(__dsub_rn(s[a] > 0 ? hi : lo, u0[a]), w[a]);
    if (ta > t_in) { t_in = ta; in_axis = a; }
    t_out_grid = fmin(t_out_grid, tb);
  }
  const double t0 = fmax(near_t, t_in), t1 = fmin(far_t, t_out_grid);
  ok = ok && t0 <= t1;
  float t_hit = INFINITY;
  int16_t l_hit = -1;
  int32_t v_hit = -1;
  double nrm[3] = {0.0, 0.0, 0.0};
  if (ok) {
    int q[3];
    double tn[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double u = __dadd_rn(u0[a], __dmul_rn(t0, w[a]));
      q[a] = (int)fmin(fmax(floor(__dadd_rn(u, 0.5)), 0.0), (double)(dim - 1));
      tn[a] = w[a] != 0.0 ? boundary(q[a], s[a], u0[a], w[a]) : INFINITY;
    }
    double t_entry = t0;
    int e_axis = t_in >= near_t ? in_axis : -1;   // the face the current voxel was entered by (-1: the ray starts inside it)
    const int max_steps = 3 * dim + 3;
    for (int it = 0; it < max_steps; ++it) {
      const int64_t p = ((int64_t)q[0] * dim + q[1]) * dim + q[2];
      if (solid_at(g, occ, labels, p)) {
        t_hit = __double2float_rn(__dadd_rn(fmax(t0, t_entry), 0.0));   // + 0: a zero time is +0
        l_hit = labels[p];
        v_hit = (int32_t)p;
        if (normal_out) {
          // -inv^T grad(occ) at q: central differences, one-sided at the grid's faces
          double gr[3];
#pragma unroll
          for (int a = 0; a < 3; ++a) {
            const int64_t st = a == 0 ? (int64_t)dim * dim : (a == 1 ? dim : 1);
            const bool has_lo = q[a] > 0, has_hi = q[a] < dim - 1;
            const double up = has_hi ? (double)occ[p + st] : (double)occ[p];
            const double dn = has_lo ? (double)occ[p - st] : (double)occ[p];
            gr[a] = has_lo && has_hi ? __dmul_rn(__dsub_rn(up, dn), 0.5) : __dsub_rn(up, dn);
          }
          double nn = normal_from(g.inv, gr, nrm);
          if (!(nn > 0.0) || !isfinite(nn)) {
            // the entry face's normal -s e_a in the network frame (inv^T of it), or -d for a ray that starts inside the voxel
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              const double f = e_axis == c ? (double)s[c] : 0.0;
              gr[c] = e_axis >= 0 ? f : 0.0;
            }
            if (e_axis >= 0) {
              nn = normal_from(g.inv, gr, nrm);
            } else {
#pragma unroll
              for (int c = 0; c < 3; ++c) nrm[c] = -(double)d[c];
              nn = __dadd_rn(__dadd_rn(__dmul_rn(nrm[0], nrm[0]), __dmul_rn(nrm[1], nrm[1])), __dmul_rn(nrm[2], nrm[2]));
            }
          }
          const double rn = __ddiv_rn(1.0, __dsqrt_rn(nn));
#pragma unroll
          for (int c = 0; c < 3; ++c) nrm[c] = __dmul_rn(nrm[c], rn);
        }
        break;
      }
      // the flat step: the axis whose boundary comes first, ties i before j before k
      int a = 0;
      if (before(tn[1], 1, tn[0], 0)) a = 1;
      if (before(tn[2], 2, pick(a, tn), a)) a = 2;
      const double ta = pick(a, tn);
      if (!(ta <= t1)) break;
      bool out = false;
#pragma unroll
      for (int c = 0; c < 3; ++c)
        if (c == a) {
          q[c] += s[c];
          out = q[c] < 0 || q[c] >= dim;
          tn[c] = boundary(q[c], s[c], u0[c], w[c]);
        }
      if (out) break;
      t_entry = ta;
      e_axis = a;
    }
  }
  t_out[r] = t_hit;
  label_out[r] = l_hit;
  voxel_out[r] = v_hit;
  if (normal_out) {
#pragma unroll
    for (int c = 0; c < 3; ++c) normal_out[3 * r + c] = __double2float_rn(nrm[c]);
  }
}

}  // namespace

int grid_cast(const float* occ, const int16_t* labels, int dim, float level, const double* T16, const double* ext3,
              const uint32_t* keep_host, const float* rays_o, const float* rays_d, int64_t n, float near_t,
              float far_t, float* t_out, int16_t* label_out, int32_t* voxel_out, float* normal_out, cudaStream_t st) {
  const char* who = "grid_cast";
  DMN_CHECK(occ != nullptr && labels != nullptr, "%s: occ and labels must not be NULL", who);
  DMN_CHECK(T16 != nullptr && ext3 != nullptr, "%s: transform and extents must not be NULL", who);
  DMN_CHECK(dim >= 2 && dim <= REGION_MAX_DIM, "%s: dim %d out of range [2, %d]", who, dim, REGION_MAX_DIM);
  DMN_CHECK(std::isfinite(level), "%s: level %g is not finite", who, (double)level);
  DMN_CHECK(std::isfinite(near_t) && std::isfinite(far_t), "%s: near %g and far %g must be finite", who, (double)near_t,
            (double)far_t);
  DMN_CHECK(near_t <= far_t, "%s: near %g > far %g", who, (double)near_t, (double)far_t);
  DMN_CHECK(n >= 0, "%s: n %lld < 0", who, (long long)n);
  DMN_CHECK(n == 0 || (rays_o && rays_d && t_out && label_out && voxel_out), "%s: a ray or output pointer is NULL", who);
  for (int k = 0; k < 16; ++k) DMN_CHECK(std::isfinite(T16[k]), "%s: the scene transform is not finite", who);
  const double* T = T16;
  const double det = T[0] * (T[5] * T[10] - T[6] * T[9]) - T[1] * (T[4] * T[10] - T[6] * T[8]) + T[2] * (T[4] * T[9] - T[5] * T[8]);
  DMN_CHECK(det > 0.0, "%s: the scene transform has det %g <= 0", who, det);
  for (int a = 0; a < 3; ++a) DMN_CHECK(ext3[a] > 0.0 && std::isfinite(ext3[a]), "%s: extents must be finite and > 0", who);
  if (n == 0) return 0;
  CastGrid g;
  grid_index_map(T16, ext3, dim, g.inv, g.b);
  g.dim = dim;
  g.level = level;
  g.masked = keep_host != nullptr;
  for (int w = 0; w < 4; ++w) g.keep.w[w] = keep_host ? keep_host[w] : ~0u;
  grid_cast_kernel<<<(unsigned)((n + CAST_THREADS - 1) / CAST_THREADS), CAST_THREADS, 0, st>>>(occ, labels, g, rays_o, rays_d, n,
                                                                                                (double)near_t, (double)far_t, t_out,
                                                                                                label_out, voxel_out, normal_out);
  DMN_LAUNCH_OK();
  return 0;
}

}  // namespace dmnerf
