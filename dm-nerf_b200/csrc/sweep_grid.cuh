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
__device__ __forceinline__ bool edit_target(const double* trans, const double* inv, const double* b, const double* lo,
                                            const double* hi, bool in, const float p[3], float t[3], double q[3]) {
  double dt[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double* r = trans + 4 * a;
    const double v = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(r[0], (double)p[0]), __dmul_rn(r[1], (double)p[1])),
                                         __dmul_rn(r[2], (double)p[2])), r[3]);
    t[a] = __double2float_rn(v);
    dt[a] = __dsub_rn((double)t[a], b[a]);
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double* row = inv + 3 * a;
    const double u = __dadd_rn(__dadd_rn(__dmul_rn(row[0], dt[0]), __dmul_rn(row[1], dt[1])), __dmul_rn(row[2], dt[2]));
    q[a] = rint(u);
    in = in && q[a] >= lo[a] && q[a] <= hi[a];
  }
  return in;
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
