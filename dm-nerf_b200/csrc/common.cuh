// Shared declarations for libdmnerf_b200.so (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <string>

#include "../../include/dmnerf_b200.h"

namespace dmnerf {

// Layer indices in reference state_dict order (networks/dm_nerf.py:65-78).
enum Layer {
  L_TRUNK0 = 0,  // mlps.0 .. mlps.7 -> 0..7
  L_RGB_FEAT = 8,
  L_INS_FEAT = 9,
  L_RGB_HID = 10,   // rgb_feature_linears.0  (128 x 283)
  L_INS_HID = 11,   // ins_feature_linears.0  (128 x 256)
  L_DENSITY = 12,
  L_INS_OUT = 13,
  L_RGB_OUT = 14,
  N_LAYERS = 15
};

constexpr int W_HID = 256;
constexpr int CH_POS = DMNERF_CH_POS;   // 63
constexpr int CH_DIR = DMNERF_CH_DIR;   // 27
constexpr int CH_IN = CH_POS + CH_DIR;  // 90
constexpr int L_POS = 10;
constexpr int L_DIR = 4;

// Live (caller-owned) fp32 parameter storage of one DM_NeRF.
struct NetParams {
  const float* w[N_LAYERS];
  const float* b[N_LAYERS];
  int ins_num;
  bool bound;
};

__host__ __device__ inline int layer_out(int l, int ins_num) {
  return l < 10 ? W_HID : (l < 12 ? W_HID / 2 : (l == L_DENSITY ? 1 : (l == L_INS_OUT ? ins_num + 1 : 3)));
}
__host__ __device__ inline int layer_in(int l) {
  return l == 0 ? CH_POS : (l == 5 ? W_HID + CH_POS : (l == L_RGB_HID ? W_HID + CH_DIR : (l >= L_INS_OUT ? W_HID / 2 : W_HID)));
}

// Activations saved by the training forward of one network (planes of row-major [M, width] matrices, in this order):
//   H0..H7 [M,256] (post-ReLU trunk outputs) | rgb_feat [M,256] | ins_feat [M,256] | rgb_hid [M,128] | ins_hid [M,128] | emb [90,M]
// (the embedded inputs are stored COLUMN-major, [90][M]: their writers own one row and a few columns each, so row-fastest storage
//  makes every store instruction of a warp one contiguous 128-byte line; their only readers are three narrow dW GEMMs)
// ... | bits: ReLU masks, 1 bit per unit, as 16-bit groups stored ROW-FASTEST: [10 planes][16 groups][M] uint16 (planes 0..7 =
//           H0..H7, 8 = rgb_hid, 9 = ins_hid (8 groups used); bit c of group g = unit 16 g + c is positive).  A warp (32
//           consecutive rows, one group) reads or writes 64 contiguous bytes.
constexpr int ACT_BITS_PLANES = 10, ACT_BITS_WORDS = 8, ACT_BITS_GROUPS = 16;
__host__ __device__ inline int64_t act_bits_index(int plane, int group, int64_t row, int64_t m) {
  return ((int64_t)plane * ACT_BITS_GROUPS + group) * m + row;
}
constexpr int ACT_FLOATS_PER_SAMPLE = CH_IN + 8 * W_HID + 2 * W_HID + 2 * (W_HID / 2) + ACT_BITS_PLANES * ACT_BITS_WORDS;   // 2986
struct ActPlanes {
  float* emb; float* h[8]; float* rgb_feat; float* ins_feat; float* rgb_hid; float* ins_hid; uint16_t* bits;
};
__host__ __device__ inline ActPlanes act_planes(float* base, int64_t m) {
  ActPlanes a;
  float* p = base;
  for (int l = 0; l < 8; ++l) { a.h[l] = p; p += m * W_HID; }
  a.rgb_feat = p; p += m * W_HID;
  a.ins_feat = p; p += m * W_HID;
  a.rgb_hid = p; p += m * (W_HID / 2);
  a.ins_hid = p; p += m * (W_HID / 2);
  a.emb = p; p += m * CH_IN;
  a.bits = reinterpret_cast<uint16_t*>(p);
  return a;
}

void set_error(const char* fmt, ...);

// Per-device one-time initialisation (kernel attributes are per device): true the first time it is called for the current
// device with this flag set.
struct PerDeviceOnce {
  bool done[64] = {};
  bool first() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return true;
    if (done[dev]) return false;
    done[dev] = true;
    return true;
  }
};
extern std::atomic<int64_t> g_launches;

#define DMN_CHECK(cond, ...)                   \
  do {                                         \
    if (!(cond)) {                             \
      ::dmnerf::set_error(__VA_ARGS__);        \
      return 1;                                \
    }                                          \
  } while (0)

#define DMN_CUDA(call)                                                                         \
  do {                                                                                         \
    cudaError_t e__ = (call);                                                                  \
    if (e__ != cudaSuccess) {                                                                  \
      ::dmnerf::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
      return 2;                                                                                \
    }                                                                                          \
  } while (0)

#define DMN_LAUNCH_OK()                                     \
  do {                                                      \
    ::dmnerf::g_launches.fetch_add(1);                      \
    DMN_CUDA(cudaGetLastError());                           \
  } while (0)

// ---- launchers implemented in the individual .cu files (all return 0 / non-zero status) ----
int launch_posenc(const float* x, int64_t m, int n_freqs, float* out, cudaStream_t st);
int launch_composite(const float* raw, const float* z, const float* rays_d, int64_t n, int s, int c, int keep_all,
                     float* rgb, float* weights, float* depth, float* ins, float* acc, cudaStream_t st);
int launch_sample_pdf(const float* bins, const float* weights, int64_t n, int nb, int ns, const float* u, float* out,
                      cudaStream_t st);
int launch_sort_concat(const float* a, const float* b, int64_t n, int na, int nb, float* out, cudaStream_t st);
int launch_prep_z(const float* z_in, int64_t z_stride, const float* t_rand, int64_t n, int s, float* z_out,
                  cudaStream_t st);
int launch_hier_sample(const float* z_c, const float* w_c, const float* u, int64_t n, int s, int ni, float* z_fine,
                       cudaStream_t st);
int launch_rays(const float* K9, const float* c2w12, int H, int W, float* rays_o, float* rays_d, cudaStream_t st);
int launch_rays_at(const float* K9, const float* c2w12, const float* c2w_dev, int64_t c2w_ld, int H, int W, const int64_t* pix,
                   int64_t n, float* rays_o, float* rays_d, cudaStream_t st);
int launch_select_pixels(uint64_t seed, int H, int W, int64_t n, int64_t* pix, cudaStream_t st);
// MLP, SIMT fp32 path.  Exactly one of x / (rays_o, rays_d, z) is used.
int launch_mlp_simt(const NetParams& p, const float* x, const float* rays_o, const float* rays_d, const float* z,
                    int64_t m, int s, float* out, float* acts, cudaStream_t st);
// Backward (backward.cu)
int launch_composite_backward(const float* raw, const float* z, const float* rays_d, int64_t n, int s, int c, int keep_all,
                              const float* g_rgb, const float* g_depth, const float* g_acc, const float* g_ins,
                              const float* g_weights, float* d_raw, int accumulate, cudaStream_t st);
// feats_missing != 0: the forward that filled `acts` did not materialise rgb_feat / ins_feat (tensor-core kernel, folded
// heads); the backward recomputes those two planes from h7 first.
struct UmmaWeights;
int launch_mlp_backward(const NetParams& p, const UmmaWeights* packed, float* acts, const float* d_out, int64_t m, float* const* grads,
                        float* scratch, int feats_missing, cudaStream_t st);
// Gradient chain (bwd_chain.cu)
int launch_mask_bits(float* acts, int64_t m, cudaStream_t st);
int launch_bwd_heads(const NetParams& p, const float* d_out, int64_t m, const uint16_t* bits, float* s12, cudaStream_t st);
int launch_bwd_chain(const UmmaWeights& w, const NetParams& p, const float* s1, const float* d_out, const ActPlanes& ap, int64_t m,
                     float* const* dy, cudaStream_t st);
size_t mlp_backward_scratch_floats(int64_t m);

// Tensor-core GEMMs of the backward (gemm_umma.cu): split-bf16 three-pass wgmma kernels for the wide layer shapes.
bool gemm_nn_tc_supported(int N, int K, int ldc, const float* C, const float* mask);
bool gemm_tn_tc_supported(int N, int K);
// mask_bits: 1-bit ReLU mask of the output, [16 groups][M] uint16 (one plane of ActPlanes::bits), or NULL.
int launch_gemm_nn_tc(const float* A, int lda, const float* W, int ldw, float* C, int ldc, int64_t M, int N, int accumulate,
                      const float* mask, const float* bias, int w_kmajor, cudaStream_t st, const uint16_t* mask_bits = nullptr);
// One product of a batched dW launch (gemm_umma.cu): C[N, K] += A[M, N]^T B[M, K]; b_cm != 0: B is column-major with that column
// stride; transpose: A is the wide operand and the result goes to C[K, N].
constexpr int TN_MAX_BATCH = 8;
struct TnProblem {
  const float* A; const float* B; float* C; float* colsum;
  int64_t b_cm;
  int lda, ldb, ldc, K, transpose;
};
int launch_gemm_tn_tc_batch(const TnProblem* probs, int n, int64_t M, int N, cudaStream_t st);
int launch_gemm_tn_tc(const float* A, int lda, const float* B, int ldb, float* C, int ldc, float* colsum, int64_t M, int N, int K,
                      int transpose, cudaStream_t st, int64_t b_cm = 0);
int gemm_tc_check_status(cudaStream_t st);

// Emptiness regulariser (penalizer.cu)
int launch_penalizer_forward(const float* raw, const float* z, const float* depth, const float* rays_d, int64_t n, int s, int c,
                             float tol, float w, void* state, float* loss, cudaStream_t st);
int launch_penalizer_backward(const float* raw, const float* z, const float* depth, const float* rays_d, int64_t n, int s, int c,
                              float tol, float w, const void* state, const float* g_loss, float* d_raw, int accumulate,
                              cudaStream_t st);
size_t penalizer_state_bytes();

// Hungarian-matched instance loss (evaluator.cu)
int launch_hungarian_costs(const float* pred, const int32_t* gt_row, int64_t n, int k, float* cost_ce, float* cost_siou,
                           float* tp, float* s_sum, float* cnt, cudaStream_t st);
int launch_ins_loss_grad(const float* pred, const int32_t* gt_row, int64_t n, int k, const int32_t* row_of_col, int n_valid,
                         const int32_t* n_valid_dev, const float* tp, const float* s_sum, const float* cnt, const float* g3,
                         float* d_pred, cudaStream_t st);
int launch_label_rows(const int32_t* labels, int64_t n, int k, int32_t* gt_row, int32_t* n_valid, cudaStream_t st);
int launch_hungarian_assign(const float* cost_ce, const float* cost_siou, const float* s_sum, const int32_t* n_valid, int64_t n, int k,
                            int32_t* row_of_col, float* loss3, cudaStream_t st);
int ins_status_take();

// Mesh extraction (mesh.cu).  Transforms are row-major 4x4 float64 host arrays, extents 3 float64 host values.
struct MeshState;                 // per-context device buffers of the mesh entry points
void mesh_state_free(MeshState* s);
int launch_grid_points(const double* T16, const double* ext3, int dim, int64_t begin, int64_t count, float* pts, cudaStream_t st);
int launch_occupancy(const float* raw, int64_t n, int c, float voxel, float* occ, cudaStream_t st);
int mc_count(MeshState** s, const float* grid, int nx, int ny, int nz, float level, int64_t* counts, cudaStream_t st);
int mc_emit(MeshState* s, const float* grid, int nx, int ny, int nz, float level, float* verts, int32_t* tris, cudaStream_t st);
int launch_to_scene(const float* v, int64_t n, const double* T16, const double* ext3, int dim, float* out, cudaStream_t st);
int mesh_normals(MeshState** s, const float* v, int64_t nv, const int32_t* tris, int64_t nt, float* normals, cudaStream_t st);
int mesh_clusters(MeshState** s, const int32_t* tris, int64_t nt, int64_t nv, int32_t* cluster, int32_t* cluster_size, cudaStream_t st);
int mesh_clean(MeshState** s, const float* v, const float* nrm, int64_t nv, const int32_t* tris, int64_t nt, const int32_t* csize,
               int min_cluster, float* out_v, float* out_n, int32_t* out_t, int64_t* counts, cudaStream_t st);
int launch_label_rays(const float* v, const float* nrm, int64_t n, float near_z, float* ro, float* rd, cudaStream_t st);
int launch_argmax_rows(const float* x, int64_t n, int c, int64_t* out, cudaStream_t st);

}  // namespace dmnerf
