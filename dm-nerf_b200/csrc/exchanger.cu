// Per-sample exchange of network outputs between the original and the transformed ("target") rays of an object edit:
// exchanger, networks/manipulator.py:18-83.  Purely element-wise over (ray, sample): one thread per sample walks the list
// of moved labels, exactly in the reference's order of updates.  HBM-streaming (reads C floats per sample per operand,
// rewrites the original's C floats when a swap happens).
//
// Moving pieces (DESIGN.md, "Moving pieces"): a move may carry a region, so that only the samples of its label inside that
// piece move.  The instance with pieces tests each sample's point against the region with region_drops (the render kernels'
// look-up) and each ray's accumulated label against its piece vote (piece_vote_kernel: the weight of the label's samples in the
// piece against the weight outside it, on the first fine pass).
#include <cstdint>
#include <cstring>

#include "common.cuh"
#include "ray_ops.cuh"

namespace dmnerf {

constexpr int EX_MAX_MOVES = DMNERF_MAX_MOVES;

struct ExchangeArgs {
  float* ori_raw;                        // [N,S,C] edited in place
  const float* tar_raw[EX_MAX_MOVES];    // [N,S,C] each
  const float* ori_acc;                  // [N,K]   rendered (post-sigmoid) instance map of the original rays, K = C - 4
  const float* tar_acc[EX_MAX_MOVES];    // [N,K]
  int move[EX_MAX_MOVES];
  int n_moves;
  int64_t total;                         // N * S
  int s, c;
  int64_t* ori_label;                    // [N,S] out: per-sample label of the original (after the occlusion fixes)
  int64_t* tar_label;                    // [N,S] out: per-sample label of the LAST target (after its occlusion fix)
};

// The pieces of an exchange: per move a region (bits == NULL: the whole label moves), the rest policy and the two per-ray votes;
// the rays and this pass's depths of the original and of every target, for the sample points.
struct PieceArgs {
  Region region[EX_MAX_MOVES];
  int rest_drop[EX_MAX_MOVES];
  const uint8_t* ori_vote[EX_MAX_MOVES];   // [N]
  const uint8_t* tar_vote[EX_MAX_MOVES];   // [N]
  const float* ori_o; const float* ori_d; const float* ori_z;                                     // [N,3] [N,3] [N,S]
  const float* tar_o[EX_MAX_MOVES]; const float* tar_d[EX_MAX_MOVES]; const float* tar_z[EX_MAX_MOVES];
};

// Is a sample of label l part of the moving piece of move (mv, r)?  A label copied from the ray's accumulated label carries the
// ray's vote, any other is judged by its point.
__device__ __forceinline__ bool piece_moving(const Region& r, int mv, int l, bool from_acc, const float* p, bool vote) {
  return l == mv && (r.bits == nullptr || (from_acc ? vote : !region_drops(r, mv, p[0], p[1], p[2])));
}

template <bool PIECES>
__global__ void exchanger_kernel(const ExchangeArgs a, const PieceArgs pc) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= a.total) return;
  const int64_t ray = idx / a.s;
  const int K = a.c - 4;
  float* o = a.ori_raw + idx * a.c;
  int ori_label = argmax_sigmoid(o + 4, K);                                     // :19-21
  const int ori_acc = argmax_sigmoid(a.ori_acc + ray * K, K - 1);               // :23-26 (last class dropped)
  int tar_label = 0;
  if constexpr (!PIECES) {
    for (int i = 0; i < a.n_moves; ++i) {
      const int mv = a.move[i];
      const float* t = a.tar_raw[i] + idx * a.c;
      if (ori_label == mv && ori_acc != mv) ori_label = ori_acc;                  // :33-36
      const bool filling = (ori_acc == mv) && (ori_label != mv);                  // :40-42
      tar_label = argmax_sigmoid(t + 4, K);                                       // :45-47
      const int tar_acc = argmax_sigmoid(a.tar_acc[i] + ray * K, K - 1);          // :50-53
      if (tar_label == mv && tar_acc != mv) tar_label = tar_acc;                  // :57-60
      const bool ori_is = ori_label == mv, tar_is = tar_label == mv;              // :64-75
      if (filling || tar_is) {                                                    // :78, :81  take the target's sample
        for (int k = 0; k < a.c; ++k) o[k] = t[k];
      } else if (ori_is) {                                                        // :82      the object moved away: empty
        for (int k = 0; k < a.c; ++k) o[k] = o[k] * 0.0f;
      }
    }
  } else {
    float po[3];
    ray_point(pc.ori_o + 3 * ray, pc.ori_d + 3 * ray, pc.ori_z[idx], po);
    bool ori_from_acc = false;
    for (int i = 0; i < a.n_moves; ++i) {
      const int mv = a.move[i];
      const Region& r = pc.region[i];
      const float* t = a.tar_raw[i] + idx * a.c;
      const bool has = r.bits != nullptr;
      const bool ori_vote = !has || pc.ori_vote[i][ray] != 0;
      const bool ori_acc_mv = ori_acc == mv && ori_vote;
      if (piece_moving(r, mv, ori_label, ori_from_acc, po, ori_vote) && !ori_acc_mv) {       // occlusion fix
        ori_label = ori_acc;
        ori_from_acc = true;
      }
      const bool ori_mv = piece_moving(r, mv, ori_label, ori_from_acc, po, ori_vote);
      const bool filling = ori_acc_mv && !ori_mv;
      tar_label = argmax_sigmoid(t + 4, K);
      const int tar_acc = argmax_sigmoid(a.tar_acc[i] + ray * K, K - 1);
      const bool tar_vote = !has || pc.tar_vote[i][ray] != 0;
      const bool tar_acc_mv = tar_acc == mv && tar_vote;
      float pt[3] = {0.0f, 0.0f, 0.0f};
      if (has) ray_point(pc.tar_o[i] + 3 * ray, pc.tar_d[i] + 3 * ray, pc.tar_z[i][idx], pt);
      bool tar_from_acc = false;
      if (piece_moving(r, mv, tar_label, false, pt, tar_vote) && !tar_acc_mv) {
        tar_label = tar_acc;
        tar_from_acc = true;
      }
      const bool tar_mv = piece_moving(r, mv, tar_label, tar_from_acc, pt, tar_vote);
      if (filling || tar_mv) {                                                    // take the target's sample
        for (int k = 0; k < a.c; ++k) o[k] = t[k];
      } else if (ori_mv || (pc.rest_drop[i] && ori_label == mv)) {                // the piece moved away / the rest vanishes
        for (int k = 0; k < a.c; ++k) o[k] = o[k] * 0.0f;
      }
    }
  }
  a.ori_label[idx] = ori_label;
  a.tar_label[idx] = tar_label;
}

int launch_exchanger(const ExchangeArgs& a, const PieceArgs* pc, cudaStream_t st) {
  if (a.total == 0) return 0;
  const unsigned blocks = (unsigned)((a.total + 255) / 256);
  if (pc) {
    exchanger_kernel<true><<<blocks, 256, 0, st>>>(a, *pc);
  } else {
    PieceArgs none;
    memset(&none, 0, sizeof(none));
    exchanger_kernel<false><<<blocks, 256, 0, st>>>(a, none);
  }
  DMN_LAUNCH_OK();
  return 0;
}

// ---- piece votes ---------------------------------------------------------------------------------------------------------
// One warp per ray, one lane per sample of a 32-sample chunk.  Per move: in = sum of w_s over the samples labelled mv whose point
// the region keeps, out = the same over those it drops, each added in ascending sample order in fp32 (a sample that does not
// count adds nothing: the sum is the sequential fp32 sum of the counted weights).  vote = in >= out.
constexpr int VOTE_WARPS = 8;

struct VoteArgs {
  const float* raw; const float* z; const float* w; const float* rays_o; const float* rays_d;
  int64_t n;
  int s, c, n_moves;
  int move[EX_MAX_MOVES];
  Region region[EX_MAX_MOVES];
  uint8_t* votes;                            // [n_moves, N]
};

__global__ void __launch_bounds__(VOTE_WARPS * 32) piece_vote_kernel(const VoteArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t ray = (int64_t)blockIdx.x * VOTE_WARPS + (threadIdx.x >> 5);
  if (ray >= a.n) return;                                                       // warp-uniform
  const int K = a.c - 4;
  float in[EX_MAX_MOVES], out[EX_MAX_MOVES];
#pragma unroll
  for (int i = 0; i < EX_MAX_MOVES; ++i) in[i] = out[i] = 0.0f;
  for (int base = 0; base < a.s; base += 32) {
    const int s = base + lane;
    int label = -1;
    float w = 0.0f, p[3] = {0.0f, 0.0f, 0.0f};
    if (s < a.s) {
      const int64_t q = ray * a.s + s;
      label = argmax_sigmoid(a.raw + q * a.c + 4, K);
      w = a.w[q];
      ray_point(a.rays_o + 3 * ray, a.rays_d + 3 * ray, a.z[q], p);
    }
    const int n_lanes = min(32, a.s - base);
#pragma unroll
    for (int i = 0; i < EX_MAX_MOVES; ++i) {
      if (i >= a.n_moves) break;
      const Region& r = a.region[i];
      const int mv = a.move[i];
      bool is_in = false, is_out = false;
      if (r.bits != nullptr && label == mv) {
        const bool drops = region_drops(r, mv, p[0], p[1], p[2]);
        is_in = !drops;
        is_out = drops;
      }
      const float w_in = is_in ? w : 0.0f, w_out = is_out ? w : 0.0f;
      for (int j = 0; j < n_lanes; ++j) {                                       // ascending sample order
        in[i] = __fadd_rn(in[i], __shfl_sync(FULL, w_in, j));
        out[i] = __fadd_rn(out[i], __shfl_sync(FULL, w_out, j));
      }
    }
  }
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < EX_MAX_MOVES; ++i)
      if (i < a.n_moves) a.votes[(int64_t)i * a.n + ray] = in[i] >= out[i] ? 1 : 0;
  }
}

// The region of a move (bits NULL: none), checked: dim and map, the moved label among the labels it applies to.
int piece_region(const dmnerf_region& d, int mv, Region& r, const char* who, int i) {
  r = Region{};
  if (!d.bits) return 0;
  if (region_from_abi(d, r, who)) return 1;
  DMN_CHECK(mv >= 0 && mv <= DMNERF_MAX_INS && obj_kept(r.applies, mv),
            "%s: move %d: moved label %d is not among the labels its region applies to", who, i, mv);
  return 0;
}

}  // namespace dmnerf

using namespace dmnerf;

extern "C" DMNERF_API int dmnerf_exchanger(float* ori_raw, const float* const* tar_raws, const float* ori_acc,
                                           const float* const* tar_accs, const int* move_labels, int n_moves, int64_t n, int s,
                                           int c, int64_t* ori_label, int64_t* tar_label, const dmnerf_pieces* pieces,
                                           void* stream) {
  DMN_CHECK(n >= 0 && s >= 1 && c > 5, "exchanger: bad sizes n=%lld s=%d c=%d", (long long)n, s, c);
  DMN_CHECK(n_moves >= 1 && n_moves <= EX_MAX_MOVES, "exchanger: between 1 and %d moved labels are supported, got %d", EX_MAX_MOVES,
            n_moves);
  DMN_CHECK(ori_raw && tar_raws && ori_acc && tar_accs && move_labels && ori_label && tar_label, "exchanger: NULL argument");
  ExchangeArgs a;
  memset(&a, 0, sizeof(a));
  a.ori_raw = ori_raw; a.ori_acc = ori_acc; a.n_moves = n_moves; a.total = n * s; a.s = s; a.c = c;
  a.ori_label = ori_label; a.tar_label = tar_label;
  for (int i = 0; i < n_moves; ++i) {
    DMN_CHECK(tar_raws[i] && tar_accs[i], "exchanger: NULL target buffer %d", i);
    a.tar_raw[i] = tar_raws[i]; a.tar_acc[i] = tar_accs[i]; a.move[i] = move_labels[i];
  }
  if (!pieces) return launch_exchanger(a, nullptr, (cudaStream_t)stream);
  PieceArgs pc;
  memset(&pc, 0, sizeof(pc));
  bool any = false;
  for (int i = 0; i < n_moves; ++i) {
    if (piece_region(pieces->region[i], a.move[i], pc.region[i], "exchanger", i)) return 1;
    if (!pc.region[i].bits) continue;
    any = true;
    DMN_CHECK(pieces->ori_vote[i] && pieces->tar_vote[i], "exchanger: move %d has a region but a NULL vote array", i);
    DMN_CHECK(pieces->tar_rays_o[i] && pieces->tar_rays_d[i] && pieces->tar_z[i],
              "exchanger: move %d has a region but NULL target rays / depths", i);
    pc.rest_drop[i] = pieces->rest_drop[i] ? 1 : 0;
    pc.ori_vote[i] = pieces->ori_vote[i]; pc.tar_vote[i] = pieces->tar_vote[i];
    pc.tar_o[i] = pieces->tar_rays_o[i]; pc.tar_d[i] = pieces->tar_rays_d[i]; pc.tar_z[i] = pieces->tar_z[i];
  }
  if (!any) return launch_exchanger(a, nullptr, (cudaStream_t)stream);
  DMN_CHECK(pieces->ori_rays_o && pieces->ori_rays_d && pieces->ori_z, "exchanger: a region needs the original rays and depths");
  pc.ori_o = pieces->ori_rays_o; pc.ori_d = pieces->ori_rays_d; pc.ori_z = pieces->ori_z;
  return launch_exchanger(a, &pc, (cudaStream_t)stream);
}

extern "C" DMNERF_API int dmnerf_piece_vote(const float* raw, const float* z, const float* weights, const float* rays_o,
                                            const float* rays_d, int64_t n, int s, int c, const int* move_labels,
                                            const dmnerf_region* regions, int n_moves, uint8_t* votes, void* stream) {
  const char* who = "piece_vote";
  DMN_CHECK(n >= 0 && s >= 1 && c > 5, "%s: bad sizes n=%lld s=%d c=%d", who, (long long)n, s, c);
  DMN_CHECK(n_moves >= 1 && n_moves <= EX_MAX_MOVES, "%s: between 1 and %d moves are supported, got %d", who, EX_MAX_MOVES, n_moves);
  DMN_CHECK(move_labels && regions && votes, "%s: NULL moves / regions / votes", who);
  DMN_CHECK(n == 0 || (raw && z && weights && rays_o && rays_d), "%s: NULL raw / depths / weights / rays", who);
  VoteArgs a;
  memset(&a, 0, sizeof(a));
  a.raw = raw; a.z = z; a.w = weights; a.rays_o = rays_o; a.rays_d = rays_d;
  a.n = n; a.s = s; a.c = c; a.n_moves = n_moves; a.votes = votes;
  for (int i = 0; i < n_moves; ++i) {
    a.move[i] = move_labels[i];
    if (piece_region(regions[i], move_labels[i], a.region[i], who, i)) return 1;
  }
  if (n == 0) return 0;
  piece_vote_kernel<<<(unsigned)((n + VOTE_WARPS - 1) / VOTE_WARPS), VOTE_WARPS * 32, 0, (cudaStream_t)stream>>>(a);
  DMN_LAUNCH_OK();
  return 0;
}
