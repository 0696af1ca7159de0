// Per-sample exchange of network outputs between the original and the transformed ("target") rays of an object edit:
// exchanger, networks/manipulator.py:18-83.  Purely element-wise over (ray, sample): one thread per sample walks the list
// of moved labels, exactly in the reference's order of updates.  HBM-streaming (reads C floats per sample per operand,
// rewrites the original's C floats when a swap happens).
#include <cstdint>
#include <cstring>

#include "common.cuh"
#include "ray_ops.cuh"

namespace dmnerf {

constexpr int EX_MAX_MOVES = 8;

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

__global__ void exchanger_kernel(const ExchangeArgs a) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= a.total) return;
  const int64_t ray = idx / a.s;
  const int K = a.c - 4;
  float* o = a.ori_raw + idx * a.c;
  int ori_label = argmax_sigmoid(o + 4, K);                                     // :19-21
  const int ori_acc = argmax_sigmoid(a.ori_acc + ray * K, K - 1);               // :23-26 (last class dropped)
  int tar_label = 0;
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
  a.ori_label[idx] = ori_label;
  a.tar_label[idx] = tar_label;
}

int launch_exchanger(const ExchangeArgs& a, cudaStream_t st) {
  if (a.total == 0) return 0;
  exchanger_kernel<<<(unsigned)((a.total + 255) / 256), 256, 0, st>>>(a);
  DMN_LAUNCH_OK();
  return 0;
}

}  // namespace dmnerf

using namespace dmnerf;

extern "C" DMNERF_API int dmnerf_exchanger(float* ori_raw, const float* const* tar_raws, const float* ori_acc,
                                           const float* const* tar_accs, const int* move_labels, int n_moves, int64_t n, int s,
                                           int c, int64_t* ori_label, int64_t* tar_label, void* stream) {
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
  return launch_exchanger(a, (cudaStream_t)stream);
}
