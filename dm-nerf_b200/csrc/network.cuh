// One network slot of a context (dmnerf_ctx::net): the caller's parameters, the tensor-core (wgmma) images packed from them
// and the error word of every launch through them.
#pragma once
#include "common.cuh"

namespace dmnerf {
namespace uk {

// The 64-wide weight chunks the consumer issues per tile, in this order: trunk layers 0..7, two half-steps each (layer 0:
// the position embedding; layers 1..7: the four activation chunks, then at layer 5 the position embedding again), then the
// heads: the folded instance hidden layer (four activation chunks), the folded colour hidden layer (four activation chunks,
// then the direction embedding) and the instance head (two activation chunks).  weight_chunks() (mlp_umma.cu) lists them for
// the producer and the packer and is checked against these counts.
constexpr int HEAD_CHUNK = 2 * (1 + 7 * 4 + 1);             // 60: the first chunk of the heads
constexpr int TILE_CHUNKS = HEAD_CHUNK + 4 + (4 + 1) + 2;   // 71
constexpr int MAX_STAGES = 2 * TILE_CHUNKS;                // the exact stream: a W_hi and a W_lo stage per chunk

// The weight stream of one image, derived from weight_chunks() by make_program: all the kernel reads of it.
struct Program {
  uint32_t stage_off[MAX_STAGES + 1];  // byte offset of every weight stage in the image; stage_off[n_stages] = image size
  int32_t n_stages;
  int32_t head_stage;                  // first stage of the heads: a tile without heads streams the stages below it
  int32_t ins_num;
};

}  // namespace uk

// One int32 in mapped host memory, readable by the host without a synchronisation and written by kernels through its device
// alias.  Allocated on first use, freed with its owner.
class MappedWord {
 public:
  MappedWord() = default;
  MappedWord(const MappedWord&) = delete;
  MappedWord& operator=(const MappedWord&) = delete;
  ~MappedWord() { if (host_) cudaFreeHost((void*)host_); }
  int init() {
    if (!host_) {
      void* h = nullptr;
      DMN_CUDA(cudaHostAlloc(&h, sizeof(int32_t), cudaHostAllocMapped));
      host_ = static_cast<volatile int32_t*>(h);
      *host_ = 0;
    }
    if (!dev_) DMN_CUDA(cudaHostGetDevicePointer((void**)&dev_, (void*)host_, 0));
    return 0;
  }
  int32_t* device() const { return dev_; }
  int read() const { return host_ ? *host_ : 0; }
  void clear() const { if (host_) *host_ = 0; }

 private:
  volatile int32_t* host_ = nullptr;
  int32_t* dev_ = nullptr;
};

// A network of a context.  bind() packs the caller's parameters into the exact tensor-core image: every layer's weight matrix
// split into bf16 hi/lo parts and laid out in the shared-memory image (K-major, 128B swizzle, 64-wide K slabs) the kernel
// streams with bulk async copies.  The network is bound, and every entry point may use it, only once that pack has succeeded.
struct Network {
  NetParams p = {};                 // the caller's live fp32 parameters (state_dict order) and ins_num
  bool bound = false;               // set by bind() only
  bool f16_ready = false;           // image16 holds the weights of the last bind (pack_f16)
  uk::Program prog = {};            // the stream of image
  uk::Program prog16 = {};          // the stream of image16: one stage per chunk
  DeviceBuffer image;               // packed bf16 operand image
  DeviceBuffer image16;             // fp16 preview network: packed fp16 image, built on first use after every bind
  DeviceBuffer bias;                // packed fp32 biases and CUDA-core layers
  DeviceBuffer fold_w_rgb;          // [128][283]: W_rgb_hid[:, :256] W_rgb_feat | W_rgb_hid[:, 256:] (the backward reads it too)
  DeviceBuffer fold_w_ins, fold_b;  // [128][256] and the two folded bias rows
  DeviceBuffer entries, pack_flag;  // the packer's chunk table and the fp16 pack's range flag
  // The error word: a kernel (network or backward GEMM) through this network that gave up on a barrier writes its code here,
  // and the NEXT launch through it refuses to start (a stalled launch can never pass silently).  It lives as long as the
  // context: a later bind does not clear it.
  MappedWord status;

  // Bind p (checked by the caller) and pack the exact image.  Unbound until the pack has succeeded.
  int bind(const NetParams& params, cudaStream_t st);
  // Pack the fp16 image if the last bind left it stale (synchronises `st`); fails for a weight above 65504.
  int pack_f16(cudaStream_t st);
  // The error word as a new launch sees it: a protocol code, or 0 (see mlp_umma.cu).
  int launch_gate(bool f16) const;
  // After a synchronisation: whether an fp16 launch stored a value above the fp16 range, clearing that code.
  bool take_f16_range() const;
  // Synchronises `st` and fails if a kernel through this network raised a protocol error (bounded wait expired).
  int check_status(cudaStream_t st) const;
};

// x [m, 90], or rays_o / rays_d with z (rays mode) or without (points mode, one sample per row).  f16: the fp16 preview network
// (inference only; pack_f16 first).
int launch_mlp_tc(const Network& net, const float* x, const float* rays_o, const float* rays_d, const float* z, int64_t m, int s,
                  float* out, float* acts, cudaStream_t st, bool f16 = false);

// Fused whole-pipeline launch (64 + 128 samples, no raw output) of a coarse / fine pair with one ins_num: see mlp_umma.cu.
// edit: the scene edit (the selected kernel), or NULL for none (the unselected kernel).
int launch_render_tc(const Network& coarse, const Network& fine, const dmnerf_render_io* io, int64_t n, int flags, cudaStream_t st,
                     const Edit* edit, bool f16);

}  // namespace dmnerf
