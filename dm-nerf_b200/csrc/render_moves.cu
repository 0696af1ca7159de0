// Rendering moved objects per sample (DESIGN.md, "Rendering moved objects"): the moves of the edited sweep applied to the raw rows of
// one pass of the stage render, by the sweep's rule (sweep_grid.cuh), so that a render and a mesh of one edit agree.  Per move: the
// target t = trans p and view direction of every sample p = o + d z, the samples whose target lies in the move's box compacted in
// order, one points-mode network launch on them, and take / vacate in place.
#include <cmath>

#include <cub/cub.cuh>

#include "common.cuh"
#include "network.cuh"
#include "ray_ops.cuh"
#include "sweep_grid.cuh"

namespace dmnerf {

static inline unsigned blocks(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

// One thread per sample i of the pass (ray i / s): p as the network prologue computes it; its target t and whether t's nearest grid
// index is in the box (flag); whether p's own nearest index is (pin: edit_target under the identity, which gives t = p exactly); the
// target's view direction trans[:3, :3] d (fp64, one rounding per operation, rounded once to fp32) normalised by the prologue's
// own fp32 expression, since points mode embeds view directions as given.  tgt [ns, 6] = (t, direction).  DEFORM (DESIGN.md,
// "Deforming objects"): t is pulled through the deformation d and the direction is the pulled-back tangent J_D^-1 trans[:3, :3] d
// (fp64, rounded once to fp32), normalised by the same expression.
template <bool DEFORM>
__global__ void move_target_kernel(const EditMove m, const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                   const float* __restrict__ z, int64_t ns, int s, float* __restrict__ tgt, int32_t* __restrict__ flag,
                                   uint8_t* __restrict__ pin, const Deform dm) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ns) return;
  const int64_t ray = i / s;
  const float o[3] = {rays_o[3 * ray], rays_o[3 * ray + 1], rays_o[3 * ray + 2]};
  const float d[3] = {rays_d[3 * ray], rays_d[3 * ray + 1], rays_d[3 * ray + 2]};
  float p[3];
  ray_point(o, d, z[i], p);
  float t[3];
  double q[3];
  bool in = !m.empty;
  Pulled P;
  if (DEFORM)
    P = edit_target_deformed(m.trans, dm, m.inv, m.b, m.lo, m.hi, in, p, t, q);
  else
    in = edit_target(m.trans, m.inv, m.b, m.lo, m.hi, in, p, t, q);
  const double identity[12] = {1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0};
  float pp[3];
  const bool p_in = edit_target(identity, m.inv, m.b, m.lo, m.hi, !m.empty, p, pp, q);
  float dt[3];
  if (DEFORM) {
    double w[3], x[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) w[a] = moved_vector(m.trans, a, d);
    deform_direction(dm, P, w, x);
#pragma unroll
    for (int a = 0; a < 3; ++a) dt[a] = __double2float_rn(x[a]);
  } else {
#pragma unroll
    for (int a = 0; a < 3; ++a) dt[a] = __double2float_rn(moved_vector(m.trans, a, d));
  }
  const float nrm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(dt[0], dt[0]), __fmul_rn(dt[1], dt[1])), __fmul_rn(dt[2], dt[2])));
  float* out = tgt + 6 * i;
  out[0] = t[0]; out[1] = t[1]; out[2] = t[2];
  out[3] = __fdiv_rn(dt[0], nrm); out[4] = __fdiv_rn(dt[1], nrm); out[5] = __fdiv_rn(dt[2], nrm);
  flag[i] = in ? 1 : 0;
  pin[i] = p_in ? 1 : 0;
}

// order-keeping compaction of the boxed targets (pos: exclusive scan of flag): points to pts [m, 3], directions to dirs [m, 3]
__global__ void move_compact_kernel(const float* __restrict__ tgt, const int32_t* __restrict__ flag, const int32_t* __restrict__ pos,
                                    int64_t ns, float* __restrict__ pts, float* __restrict__ dirs) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ns || !flag[i]) return;
  const int64_t o = pos[i];
  const float* t = tgt + 6 * i;
  pts[3 * o] = t[0]; pts[3 * o + 1] = t[1]; pts[3 * o + 2] = t[2];
  dirs[3 * o] = t[3]; dirs[3 * o + 1] = t[4]; dirs[3 * o + 2] = t[5];
}

__global__ void move_count_kernel(const int32_t* flag, const int32_t* pos, int64_t ns, int64_t* out) {
  out[0] = (int64_t)pos[ns - 1] + flag[ns - 1];
}

// One thread per sample: take the network's row at the target (all c channels), or vacate the sample (density 0, logits kept).
//   take:   t in the box && edit_takes(label(t), occ(t), group, occ_p) && (no piece || the piece keeps t for label(t));
//   vacate: otherwise label_p in group && ((the piece keeps p for label_p, every p without one) && p's index in the box
//                                          || rest_drop && the piece does not keep p).
// Unlike the sweep's vacate there is no occ_p > level test (a render composites every density, so a vacated object must leave no
// haze); the box bounds the vacate instead.  A COPY (DESIGN.md, "Copying objects") takes the same rows and never vacates.
template <bool COPY>
__global__ void move_apply_kernel(const EditMove m, const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                  const float* __restrict__ z, int64_t ns, int s, int c, float voxel, float level,
                                  const int32_t* __restrict__ flag, const int32_t* __restrict__ pos, const uint8_t* __restrict__ pin,
                                  const float* __restrict__ tgt, const float* __restrict__ traw, float* __restrict__ raw) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ns) return;
  float* r = raw + i * c;
  const bool has_piece = m.piece.bits != nullptr;
  if (flag[i]) {
    const float* rt = traw + (int64_t)pos[i] * c;
    const int lt = argmax_sigmoid(rt + 4, c - 4);
    const float* t = tgt + 6 * i;
    if (edit_takes(lt, occupancy_of(rt[3], voxel), m.group, occupancy_of(r[3], voxel), level) &&
        (!has_piece || !region_drops(m.piece, lt, t[0], t[1], t[2]))) {
      for (int k = 0; k < c; ++k) r[k] = rt[k];
      return;
    }
  }
  if (COPY) return;
  const int lp = argmax_sigmoid(r + 4, c - 4);
  if (!in_group(m.group, lp)) return;
  bool in_piece = true;
  if (has_piece) {
    const int64_t ray = i / s;
    const float o[3] = {rays_o[3 * ray], rays_o[3 * ray + 1], rays_o[3 * ray + 2]};
    const float d[3] = {rays_d[3 * ray], rays_d[3 * ray + 1], rays_d[3 * ray + 2]};
    float p[3];
    ray_point(o, d, z[i], p);
    in_piece = !region_drops(m.piece, lp, p[0], p[1], p[2]);
  }
  if (in_piece ? pin[i] != 0 : m.rest_drop != 0) r[3] = 0.0f;
}

int render_moves_pass(MovesState& s, const Network& net, bool f16, const EditMove* moves, const int32_t* copies, int n_moves,
                      const float* rays_o, const float* rays_d, const float* z, int64_t n, int s_per_ray, int c, float voxel,
                      float level, float* raw, int64_t* evaluated, cudaStream_t st, const Deform* deforms) {
  const int64_t ns = n * s_per_ray;
  if (ns == 0) return 0;
  DMN_CHECK(ns < INT32_MAX, "render_moved: %lld samples in one pass exceed the 32-bit scan", (long long)ns);
  float *tgt, *pts;
  int32_t *flag, *pos;
  uint8_t* pin;
  int64_t* tot;
  if (s.tgt.get((size_t)ns * 6, &tgt) || s.flag.get((size_t)ns, &flag) || s.pin.get((size_t)ns, &pin) ||
      s.pos.get((size_t)ns, &pos) || s.pts.get((size_t)ns * 6, &pts) || s.total.get(1, &tot))
    return 2;
  float* dirs = pts + (size_t)ns * 3;
  size_t temp_bytes = 0;
  DMN_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, temp_bytes, flag, pos, (int)ns, st));
  uint8_t* temp;
  if (s.temp.get(temp_bytes, &temp)) return 2;
  for (int i = 0; i < n_moves; ++i) {
    const EditMove& m = moves[i];
    if (deforms && deforms[i].n_knots)
      move_target_kernel<true><<<blocks(ns, 256), 256, 0, st>>>(m, rays_o, rays_d, z, ns, s_per_ray, tgt, flag, pin, deforms[i]);
    else
      move_target_kernel<false><<<blocks(ns, 256), 256, 0, st>>>(m, rays_o, rays_d, z, ns, s_per_ray, tgt, flag, pin, Deform{});
    DMN_LAUNCH_OK();
    DMN_CUDA(cub::DeviceScan::ExclusiveSum(temp, temp_bytes, flag, pos, (int)ns, st));
    move_count_kernel<<<1, 1, 0, st>>>(flag, pos, ns, tot);
    DMN_LAUNCH_OK();
    int64_t cnt = 0;
    DMN_CUDA(cudaMemcpyAsync(&cnt, tot, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    DMN_CUDA(cudaStreamSynchronize(st));
    float* traw = nullptr;
    if (cnt) {
      move_compact_kernel<<<blocks(ns, 256), 256, 0, st>>>(tgt, flag, pos, ns, pts, dirs);
      DMN_LAUNCH_OK();
      if (s.raw.get((size_t)cnt * c, &traw)) return 2;
      if (int rc = launch_mlp_tc(net, nullptr, pts, dirs, nullptr, cnt, 1, traw, nullptr, st, f16)) return rc;
    }
    if (copies && copies[i])
      move_apply_kernel<true><<<blocks(ns, 256), 256, 0, st>>>(m, rays_o, rays_d, z, ns, s_per_ray, c, voxel, level, flag, pos, pin, tgt,
                                                               traw, raw);
    else
      move_apply_kernel<false><<<blocks(ns, 256), 256, 0, st>>>(m, rays_o, rays_d, z, ns, s_per_ray, c, voxel, level, flag, pos, pin,
                                                                tgt, traw, raw);
    DMN_LAUNCH_OK();
    *evaluated += cnt;
  }
  return 0;
}

}  // namespace dmnerf
