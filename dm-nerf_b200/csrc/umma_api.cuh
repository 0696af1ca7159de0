// Interface between the C-ABI layer and the tensor-core (wgmma) MLP kernel.
#pragma once
#include "common.cuh"

namespace dmnerf {

// Tensor-core operand image of one DM_NeRF: every layer's weight matrix split into bf16 hi/lo parts and
// laid out in the exact shared-memory image (K-major, 128B swizzle, 64-wide K slabs) the kernel streams
// with bulk async copies.  Owned by the context; rebuilt by dmnerf_set_weights.
struct UmmaWeights {
  void* image = nullptr;        // packed bf16 operand image (device)
  float* bias = nullptr;        // packed fp32 biases (device)
  void* extra = nullptr;        // kernel program + folded-weight scratch (mlp_umma.cu)
  size_t image_bytes = 0;
  int ins_num = 0;
  bool ready = false;
};

const float* umma_fold_w_rgb(const UmmaWeights& w);      // [128][283]: W_rgb_hid[:, :256] W_rgb_feat | W_rgb_hid[:, 256:]
int32_t* umma_status_word(const UmmaWeights& w);
int umma_status_peek(const UmmaWeights& w);            // host-side read of the error word (mapped memory, no synchronisation)

int umma_weights_pack(UmmaWeights& w, const NetParams& p, cudaStream_t st);
void umma_weights_free(UmmaWeights& w);
bool umma_available(const UmmaWeights& w);
// Synchronises `st` and fails if the kernel raised a protocol error (bounded wait expired).
int umma_check_status(const UmmaWeights& w, cudaStream_t st);
int launch_mlp_umma(const UmmaWeights& w, const NetParams& p, const float* x, const float* rays_o, const float* rays_d,
                    const float* z, int64_t m, int s, float* out, float* acts, cudaStream_t st);

// Fused whole-pipeline launch (64 + 128 samples, no raw output): see mlp_umma.cu.
int launch_render_umma(const UmmaWeights& wc, const UmmaWeights& wf, const dmnerf_render_io* io, int64_t n, int flags,
                       cudaStream_t st);

}  // namespace dmnerf
