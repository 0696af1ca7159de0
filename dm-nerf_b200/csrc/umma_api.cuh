// Interface between the C-ABI layer and the tensor-core (wgmma) MLP kernel.
#pragma once
#include "common.cuh"

namespace dmnerf {

// Tensor-core operand image of one DM_NeRF: every layer's weight matrix split into bf16 hi/lo parts and
// laid out in the exact shared-memory image (K-major, 128B swizzle, 64-wide K slabs) the kernel streams
// with bulk async copies.  Owned by the context; rebuilt by dmnerf_set_weights.
struct UmmaWeights {
  uint8_t* image = nullptr;     // packed bf16 operand image (device)
  uint8_t* image16 = nullptr;   // fp16 preview network: packed fp16 image (device), built on first use after every re-pack
  float* bias = nullptr;        // packed fp32 biases (device)
  void* extra = nullptr;        // the memory behind these, kernel program, folded-weight scratch, error word (mlp_umma.cu)
  int ins_num = 0;
  bool ready = false;
  bool f16_ready = false;       // image16 holds the weights of the last umma_weights_pack
};

const float* umma_fold_w_rgb(const UmmaWeights& w);      // [128][283]: W_rgb_hid[:, :256] W_rgb_feat | W_rgb_hid[:, 256:]
// Device alias of the weight set's error word: the network kernels and the backward GEMMs through this set write their codes here.
int32_t* umma_status_word(const UmmaWeights& w);
int umma_status_peek(const UmmaWeights& w);            // host-side read of the error word (mapped memory, no synchronisation)

int umma_weights_pack(UmmaWeights& w, const NetParams& p, cudaStream_t st);
// Pack the fp16 image if the last umma_weights_pack left it stale (synchronises `st`); fails for a weight above 65504.
int umma_weights_pack_f16(UmmaWeights& w, const NetParams& p, cudaStream_t st);
void umma_weights_free(UmmaWeights& w);
bool umma_available(const UmmaWeights& w);
// Synchronises `st` and fails if a kernel through this weight set raised a protocol error (bounded wait expired).
int umma_check_status(const UmmaWeights& w, cudaStream_t st);
// After a synchronisation: whether an fp16 launch stored a value above the fp16 range, clearing that code.
bool umma_take_f16_range(const UmmaWeights& w);
// f16: the fp16 preview network (inference only; umma_weights_pack_f16 first)
int launch_mlp_umma(const UmmaWeights& w, const NetParams& p, const float* x, const float* rays_o, const float* rays_d,
                    const float* z, int64_t m, int s, float* out, float* acts, cudaStream_t st, bool f16 = false);

// Fused whole-pipeline launch (64 + 128 samples, no raw output): see mlp_umma.cu.
// edit: the scene edit (the selected kernel), or NULL for none (the unselected kernel).
int launch_render_umma(const UmmaWeights& wc, const UmmaWeights& wf, const dmnerf_render_io* io, int64_t n, int flags,
                       cudaStream_t st, const Edit* edit, bool f16);

}  // namespace dmnerf
