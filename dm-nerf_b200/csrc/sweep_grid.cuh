// The occupancy sweep's grid as the device sees it (DESIGN.md, "Mesh extraction" and "Meshing an edited scene"): its fp32 grid
// points, and the target and nearest grid index of a point under a move.  Shared by the edited sweep (mesh.cu), the collision
// checks (collide.cu) and the moved render (render_moves.cu), so that all take the same decisions.
#pragma once
#include "common.cuh"

namespace dmnerf {

struct GridXform {
  float r[12];     // rows of [R | t], float32 like the original's torch.from_numpy(transform).float()
  float s[3];      // extents / 2 (float32)
  float step;      // torch.linspace(-1, 1, dim) step
  int dim;
};

inline GridXform make_xform(const double* T16, const double* ext3, int dim) {
  GridXform g;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) g.r[4 * r + c] = (float)T16[4 * r + c];
  for (int a = 0; a < 3; ++a) g.s[a] = (float)(ext3[a] / 2.0);
  g.step = 2.0f / (float)(dim - 1);
  g.dim = dim;
  return g;
}

// The grid's index map of objects.grid_affine: p = A idx + b with A = S R diag(h), b = S (t - R e), h = extents / (dim - 1),
// e = extents / 2 and S the axis swap (x, y, z) -> (x, -z, y); inv = diag(1 / h) R^-1 S^T, R^-1 = adj(R) / det(R).
inline void grid_index_map(const double* T, const double* ext, int dim, double inv[9], double b[3]) {
  const double R[3][3] = {{T[0], T[1], T[2]}, {T[4], T[5], T[6]}, {T[8], T[9], T[10]}};
  double adj[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      const int i1 = (j + 1) % 3, i2 = (j + 2) % 3, j1 = (i + 1) % 3, j2 = (i + 2) % 3;
      adj[i][j] = R[i1][j1] * R[i2][j2] - R[i1][j2] * R[i2][j1];       // cofactor (j, i)
    }
  const double det = (R[0][0] * adj[0][0] + R[0][1] * adj[1][0]) + R[0][2] * adj[2][0];
  double w[3];
  for (int r = 0; r < 3; ++r)
    w[r] = T[4 * r + 3] - ((R[r][0] * (ext[0] / 2.0) + R[r][1] * (ext[1] / 2.0)) + R[r][2] * (ext[2] / 2.0));
  b[0] = w[0]; b[1] = -w[2]; b[2] = w[1];
  for (int a = 0; a < 3; ++a) {
    const double scale = (double)(dim - 1) / ext[a];
    const double ri[3] = {adj[a][0] / det, adj[a][1] / det, adj[a][2] / det};
    // column c of S^T: S^T e_0 = e_0, S^T e_1 = -e_2, S^T e_2 = e_1
    inv[3 * a] = scale * ri[0];
    inv[3 * a + 1] = scale * -ri[2];
    inv[3 * a + 2] = scale * ri[1];
  }
}

// torch.linspace(-1, 1, dim) on the CPU in float32: start + step * i below the half, end - step * (dim - 1 - i) above it, each a
// single rounding (fused multiply-add)
__device__ __forceinline__ float linspace_m11(int i, const GridXform& g) {
  return i < g.dim / 2 ? __fmaf_rn(g.step, (float)i, -1.0f) : __fmaf_rn(-g.step, (float)(g.dim - 1 - i), 1.0f);
}

// visualizer.make_3D_grid / grid_within_bound + mesh_generator.py:28-29, in the original's fp32 operation order:
// q = (R q_scaled summed left to right) + t, then (x, y, z) -> (x, -z, y)
__device__ __forceinline__ void sweep_point(const GridXform& g, int64_t p, float out[3]) {
  const int64_t d = g.dim;
  const float q[3] = {__fmul_rn(linspace_m11((int)(p / (d * d)), g), g.s[0]), __fmul_rn(linspace_m11((int)((p / d) % d), g), g.s[1]),
                      __fmul_rn(linspace_m11((int)(p % d), g), g.s[2])};
  float w[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const float* row = g.r + 4 * r;
    w[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(row[0], q[0]), __fmul_rn(row[1], q[1])), __fmul_rn(row[2], q[2])), row[3]);
  }
  out[0] = w[0];
  out[1] = -w[2];
  out[2] = w[1];
}

// The target of sweep point p under a move: t = trans p (row-major 3x4, fp64, rounded once to fp32), the nearest grid index
// q = rint(inv (t - b)) of t (fp64, half to even; inv and b: the grid's index map), and whether q lies in the inclusive box
// [lo, hi] (`in` false: never).  An fp32 sweep point maps to its own index, also on the grid's faces.  Every operation is rounded
// once (no contraction), so that a numpy restatement takes the same decisions.
// q = rint(inv dt) and the box test of edit_target, dt = t - b
__device__ __forceinline__ bool index_in_box(const double* inv, const double* lo, const double* hi, bool in, const double dt[3],
                                             double q[3]) {
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double* row = inv + 3 * a;
    const double u = __dadd_rn(__dadd_rn(__dmul_rn(row[0], dt[0]), __dmul_rn(row[1], dt[1])), __dmul_rn(row[2], dt[2]));
    q[a] = rint(u);
    in = in && q[a] >= lo[a] && q[a] <= hi[a];
  }
  return in;
}

// y = trans p in fp64, not rounded
__device__ __forceinline__ double moved_coord(const double* trans, int a, const float p[3]) {
  const double* r = trans + 4 * a;
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(r[0], (double)p[0]), __dmul_rn(r[1], (double)p[1])), __dmul_rn(r[2], (double)p[2])),
                   r[3]);
}

// w = trans[:3, :3] v in fp64, not rounded: the view direction of ray direction v under a move (the moved render, render_moves.cu,
// and the edit view, edit_view.cu), before a deformation pulls it back and before it is rounded to fp32
__device__ __forceinline__ double moved_vector(const double* trans, int a, const float v[3]) {
  const double* r = trans + 4 * a;
  return __dadd_rn(__dadd_rn(__dmul_rn(r[0], (double)v[0]), __dmul_rn(r[1], (double)v[1])), __dmul_rn(r[2], (double)v[2]));
}

__device__ __forceinline__ bool edit_target(const double* trans, const double* inv, const double* b, const double* lo,
                                            const double* hi, bool in, const float p[3], float t[3], double q[3]) {
  double dt[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    t[a] = __double2float_rn(moved_coord(trans, a, p));
    dt[a] = __dsub_rn((double)t[a], b[a]);
  }
  return index_in_box(inv, lo, hi, in, dt, q);
}

// ---- deformations (DESIGN.md, "Deforming objects") -------------------------------------------------------------------------
// Every expression is fp64 with one rounding per operation (the _rn intrinsics: no contraction) and nothing transcendental, so
// that oracle/deform_oracle.py takes the same decisions.

// A deformation's table at height h: the knot interval k, the interpolated A (row-major) and t, det A, and whether h lies inside
// [h0, h0 + (K - 1) dh] (the derivative in h is zero where the table is clamped).  (u, v): the pulled frame coordinates.
struct Pulled {
  double a[4], t[2], det, u, v, h;
  int k;
  bool inside;
};

// x = D^-1(y) for y in the network frame: frame coordinates (u, v, h) of y, r = (h - h0) / dh, k = clamp(floor r, 0, K - 2),
// s = clamp(r - k, 0, 1), A and t interpolated per entry as A_k + s (A_k+1 - A_k), (u', v') = adj(A) ((u, v) - t) / det A, and
// x = ((c + u' e_u) + v' e_v) + h e_h.
__device__ __forceinline__ Pulled deform_pull(const Deform& D, const double y[3], double x[3]) {
  const double *eu = D.frame, *ev = D.frame + 3, *eh = D.frame + 6, *c = D.frame + 9;
  const double d[3] = {__dsub_rn(y[0], c[0]), __dsub_rn(y[1], c[1]), __dsub_rn(y[2], c[2])};
  auto dot = [&](const double* e) {
    return __dadd_rn(__dadd_rn(__dmul_rn(e[0], d[0]), __dmul_rn(e[1], d[1])), __dmul_rn(e[2], d[2]));
  };
  const double u = dot(eu), v = dot(ev);
  Pulled P;
  P.h = dot(eh);
  const double r = __ddiv_rn(__dsub_rn(P.h, D.h0), D.dh);
  const double kf = fmin(fmax(floor(r), 0.0), (double)(D.n_knots - 2));
  P.k = (int)kf;
  P.inside = r >= 0.0 && r <= (double)(D.n_knots - 1);
  const double s = fmin(fmax(__dsub_rn(r, kf), 0.0), 1.0);
  const double* k0 = D.knots + 6 * P.k;
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    const double e = __dadd_rn(k0[j], __dmul_rn(s, __dsub_rn(k0[6 + j], k0[j])));
    if (j < 4) P.a[j] = e;
    else P.t[j - 4] = e;
  }
  P.det = __dsub_rn(__dmul_rn(P.a[0], P.a[3]), __dmul_rn(P.a[1], P.a[2]));
  const double du = __dsub_rn(u, P.t[0]), dv = __dsub_rn(v, P.t[1]);
  P.u = __ddiv_rn(__dsub_rn(__dmul_rn(P.a[3], du), __dmul_rn(P.a[1], dv)), P.det);
  P.v = __ddiv_rn(__dsub_rn(__dmul_rn(P.a[0], dv), __dmul_rn(P.a[2], du)), P.det);
#pragma unroll
  for (int a = 0; a < 3; ++a)
    x[a] = __dadd_rn(__dadd_rn(__dadd_rn(c[a], __dmul_rn(P.u, eu[a])), __dmul_rn(P.v, ev[a])), __dmul_rn(P.h, eh[a]));
  return P;
}

// edit_target of a deformed move: y = trans p (fp64, not rounded), x = D^-1(y) rounded once to fp32 as t, then the same box test.
__device__ __forceinline__ Pulled edit_target_deformed(const double* trans, const Deform& D, const double* inv, const double* b,
                                                       const double* lo, const double* hi, bool& in, const float p[3], float t[3],
                                                       double q[3]) {
  double y[3], x[3], dt[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) y[a] = moved_coord(trans, a, p);
  const Pulled P = deform_pull(D, y, x);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    t[a] = __double2float_rn(x[a]);
    dt[a] = __dsub_rn((double)t[a], b[a]);
  }
  in = index_in_box(inv, lo, hi, in, dt, q);
  return P;
}

// The pulled-back tangent J_D^-1 w of a direction w (network frame, fp64) at the pulled point P: in frame coordinates
// (w_u, w_v, w_h), g = A' (u', v') + t' (A' = (A_k+1 - A_k) / dh and t' likewise inside the knots, zero where clamped),
// r = (w_u, w_v) - w_h g, (d_u, d_v) = adj(A) r / det A, and out = (d_u e_u + d_v e_v) + w_h e_h.
__device__ __forceinline__ void deform_direction(const Deform& D, const Pulled& P, const double w[3], double out[3]) {
  const double *eu = D.frame, *ev = D.frame + 3, *eh = D.frame + 6;
  auto dot = [&](const double* e) {
    return __dadd_rn(__dadd_rn(__dmul_rn(e[0], w[0]), __dmul_rn(e[1], w[1])), __dmul_rn(e[2], w[2]));
  };
  const double wu = dot(eu), wv = dot(ev), wh = dot(eh);
  double g0 = 0.0, g1 = 0.0;
  if (P.inside) {
    const double* k0 = D.knots + 6 * P.k;
    double s[6];
#pragma unroll
    for (int j = 0; j < 6; ++j) s[j] = __ddiv_rn(__dsub_rn(k0[6 + j], k0[j]), D.dh);
    g0 = __dadd_rn(__dadd_rn(__dmul_rn(s[0], P.u), __dmul_rn(s[1], P.v)), s[4]);
    g1 = __dadd_rn(__dadd_rn(__dmul_rn(s[2], P.u), __dmul_rn(s[3], P.v)), s[5]);
  }
  const double r0 = __dsub_rn(wu, __dmul_rn(wh, g0)), r1 = __dsub_rn(wv, __dmul_rn(wh, g1));
  const double du = __ddiv_rn(__dsub_rn(__dmul_rn(P.a[3], r0), __dmul_rn(P.a[1], r1)), P.det);
  const double dv = __ddiv_rn(__dsub_rn(__dmul_rn(P.a[0], r1), __dmul_rn(P.a[2], r0)), P.det);
#pragma unroll
  for (int a = 0; a < 3; ++a) out[a] = __dadd_rn(__dadd_rn(__dmul_rn(du, eu[a]), __dmul_rn(dv, ev[a])), __dmul_rn(wh, eh[a]));
}

// mesh_generator.py:51-62: occ = 1 - exp(-relu(sigma) * voxel), sigma = channel 3 of the network output [n, c]
__device__ __forceinline__ float occupancy_of(float a, float voxel) {
  const float r = a > 0.f ? a : (a != a ? a : 0.f);           // torch.relu keeps NaN
  return __fsub_rn(1.0f, expf(__fmul_rn(-r, voxel)));
}

// The take test of a move of the labels `group` (piece aside): the target (lt, ot) holds one of them, and it is solid or the point
// it replaces (occupancy o) is not.  The moved render (render_moves.cu) calls it; edit_rule below spells the same expression out,
// because calling it there reorders the SASS of the edited sweep's and the grid-only edit's kernels.
__device__ __forceinline__ bool edit_takes(int lt, float ot, const ObjMask& group, float o, float level) {
  return in_group(group, lt) && (ot > level || o <= level);
}

// The edit rule at one grid point p (DESIGN.md, "Meshing an edited scene", "Moving objects together"), shared by the edited sweep
// (the network at the target) and the grid-only edit (collide.cu: the unedited grid at the target's nearest index).  m: the
// move's label set `group`, rest_drop and piece (taken by value, which keeps the edited sweep's SASS as it was before the rule was
// shared).  target(lt, ot) gives the label and occupancy at the target and is called only in the box; drops_target(lt) is the
// piece's region_drops at the target for the target's label and in_piece(b, l) sets b to whether the piece keeps p for p's label
// l, both called only with a piece.
//   take:   in the box && lt in group && (ot > level || o <= level) && (no piece || !drops_target(lt)): take(ot, lt) writes
//           (o, l) <- (ot, lt);
//   vacate: otherwise l in group && o > level && (no piece || p in the piece || rest_drop): vacate() writes o <- 0, the label
//           kept.  A copy (COPY, DESIGN.md, "Copying objects") takes as a move does and never vacates.
// A move of one label has group = {label}: the set tests are that label's equality tests.
template <bool COPY = false, class Move, class Target, class DropsTarget, class InPiece, class Take, class Vacate>
__device__ __forceinline__ void edit_rule(const Move m, bool in_box, const Target& target, float o, int l, float level,
                                          const DropsTarget& drops_target, const InPiece& in_piece_of, const Take& take,
                                          const Vacate& vacate) {
  const bool has_piece = m.piece.bits != nullptr;
  if (in_box) {
    int lt;
    float ot;
    target(lt, ot);
    if (in_group(m.group, lt) && (ot > level || o <= level) && (!has_piece || !drops_target(lt))) {
      take(ot, lt);
      return;
    }
  }
  if (!COPY && in_group(m.group, l) && o > level) {
    bool in_piece = true;
    if (has_piece) in_piece_of(in_piece, l);
    if (in_piece || m.rest_drop) vacate();
  }
}

}  // namespace dmnerf
