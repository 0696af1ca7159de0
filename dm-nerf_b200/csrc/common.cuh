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
};

__host__ __device__ inline int layer_out(int l, int ins_num) {
  return l < 10 ? W_HID : (l < 12 ? W_HID / 2 : (l == L_DENSITY ? 1 : (l == L_INS_OUT ? ins_num + 1 : 3)));
}
__host__ __device__ constexpr int layer_in(int l) {
  return l == 0 ? CH_POS : (l == 5 ? W_HID + CH_POS : (l == L_RGB_HID ? W_HID + CH_DIR : (l >= L_INS_OUT ? W_HID / 2 : W_HID)));
}

// Activations saved by the training forward of one network (planes of row-major [M, width] matrices, in this order):
//   H0..H7 [M,256] (post-ReLU trunk outputs) | rgb_hid [M,128] | ins_hid [M,128] | emb [90,M]
// (the embedded inputs are stored COLUMN-major, [90][M]: their writers own one row and a few columns each, so row-fastest storage
//  makes every store instruction of a warp one contiguous 128-byte line; their only readers are three narrow dW GEMMs)
// ... | bits: ReLU masks, 1 bit per unit, as 16-bit groups stored ROW-FASTEST: [10 planes][16 groups][M] uint16 (planes 0..7 =
//           H0..H7, 8 = rgb_hid, 9 = ins_hid (8 groups used); bit c of group g = unit 16 g + c is positive).  A warp (32
//           consecutive rows, one group) reads or writes 64 contiguous bytes.
constexpr int ACT_BITS_PLANES = 10, ACT_BITS_WORDS = 8, ACT_BITS_GROUPS = 16;
__host__ __device__ inline int64_t act_bits_index(int plane, int group, int64_t row, int64_t m) {
  return ((int64_t)plane * ACT_BITS_GROUPS + group) * m + row;
}
constexpr int ACT_FLOATS_PER_SAMPLE = CH_IN + 8 * W_HID + 2 * (W_HID / 2) + ACT_BITS_PLANES * ACT_BITS_WORDS;   // 2474
struct ActPlanes {
  float* emb; float* h[8]; float* rgb_hid; float* ins_hid; uint16_t* bits;
};
__host__ __device__ inline ActPlanes act_planes(float* base, int64_t m) {
  ActPlanes a;
  float* p = base;
  for (int l = 0; l < 8; ++l) { a.h[l] = p; p += m * W_HID; }
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

// Grow-only device buffer, the only owner of device memory in the library: get() returns room for n values of T, reallocating
// (contents lost) with 25 % headroom when a request outgrows it.  Every request carries a 16-byte tail, so that an empty one
// still yields a valid pointer (a NULL scratch pointer would turn a cub call into a size query).
class DeviceBuffer {
 public:
  DeviceBuffer() = default;
  DeviceBuffer(const DeviceBuffer&) = delete;
  DeviceBuffer& operator=(const DeviceBuffer&) = delete;
  ~DeviceBuffer() { if (ptr_) cudaFree(ptr_); }
  template <class T>
  int get(size_t n, T** out) {
    const size_t bytes = n * sizeof(T) + 16;
    if (bytes > cap_) {
      if (ptr_) DMN_CUDA(cudaFree(ptr_));
      ptr_ = nullptr; cap_ = 0;
      DMN_CUDA(cudaMalloc(&ptr_, bytes + bytes / 4));
      cap_ = bytes + bytes / 4;
    }
    *out = static_cast<T*>(ptr_);
    return 0;
  }
  template <class T>
  T* data() const { return static_cast<T*>(ptr_); }   // what the last get() returned

 private:
  void* ptr_ = nullptr;
  size_t cap_ = 0;
};

// Number of SMs of the current device (the grid of a persistent kernel).
inline int sm_count(int* sms) {
  int dev = 0;
  DMN_CUDA(cudaGetDevice(&dev));
  DMN_CUDA(cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev));
  return 0;
}

// Object selection (DESIGN.md, "Object selection"): the set of kept labels 0 .. ins_num as a 128-bit mask, bit k of word
// k / 32.  A sample whose arg-max label (argmax_sigmoid, ray_ops.cuh) is not kept has alpha = 0 in the composite.
struct ObjMask {
  uint32_t w[4];
};
__host__ __device__ inline bool obj_kept(const ObjMask& m, int label) {
  const uint32_t word = label < 64 ? (label < 32 ? m.w[0] : m.w[1]) : (label < 96 ? m.w[2] : m.w[3]);   // no dynamic indexing
  return (word >> (label & 31)) & 1u;
}

// Region selection (DESIGN.md, "Region selection"): one bit per point of a sweep grid [dim]^3 (C order, bit v & 31 of word
// v >> 5), the fp32 voxel map [M | c] (row-major 3x4) from the network frame to grid indices, and the rule's two settings: the
// labels it applies to and what happens to a sample outside the grid.  bits == NULL: no region.  The per-sample test is
// region_drops (ray_ops.cuh).
constexpr int REGION_MAX_DIM = 1290;                          // dim^3 < 2^31, as the component grids
struct Region {
  const uint32_t* bits;
  float map[12];
  int32_t dim;
  int32_t outside_keep;        // 1: a sample outside the grid is kept; 0: dropped
  ObjMask applies;             // labels the region applies to
};
inline int64_t region_words(int dim) { return ((int64_t)dim * dim * dim + 31) / 32; }

// Object appearance (DESIGN.md, "Object appearance"): one row per label 0 .. ins_num of APPEARANCE_ROW floats, the colour map
// [M | b] (row-major 3x4), the density scale and 3 floats of padding (a row is 4 aligned float4).  The per-sample step is
// appearance_apply (ray_ops.cuh).
constexpr int APPEARANCE_ROW = 16;

// The scene edit of a render call, checked (abi.cu scene_edit): the kept labels (every label when the caller gave no selection),
// the region (bits == NULL: none) and the appearance table (device, ins_num + 1 rows, or NULL: none).  A launcher given an Edit
// runs the selected kernels; given NULL, the unselected ones.
struct Edit {
  ObjMask keep;
  Region region;
  const float* appearance;
};

// ---- launchers implemented in the individual .cu files (all return 0 / non-zero status) ----
int launch_posenc(const float* x, int64_t m, int n_freqs, float* out, cudaStream_t st);
// edit: the scene edit (the selected kernel; a region needs rays_o), or NULL for none (the unselected kernel).
int launch_composite(const float* raw, const float* z, const float* rays_d, int64_t n, int s, int c, int keep_all,
                     float* rgb, float* weights, float* depth, float* ins, float* acc, cudaStream_t st,
                     const Edit* edit = nullptr, const float* rays_o = nullptr);
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
// flags: bit 0 = the forward that filled `acts` wrote the ReLU bit planes (tensor-core kernel; otherwise the backward derives
// them from the saved activations first), bit 1 = grads are already zero.  wimage / partial: the scratch of the tensor-core
// GEMMs (launch_gemm_nn_tc / launch_gemm_tn_tc_batch).
struct Network;
int launch_mlp_backward(const Network& net, float* acts, const float* d_out, int64_t m, float* const* grads, float* scratch, int flags,
                        DeviceBuffer& wimage, DeviceBuffer& partial, cudaStream_t st);
// Gradient chain (bwd_chain.cu)
int launch_mask_bits(float* acts, int64_t m, cudaStream_t st);
int launch_bwd_heads(const NetParams& p, const float* d_out, int64_t m, const uint16_t* bits, float* s12, cudaStream_t st);
int launch_bwd_chain(const Network& net, const float* s1, const float* d_out, const ActPlanes& ap, int64_t m, float* const* dy,
                     DeviceBuffer& wimage, cudaStream_t st);
size_t mlp_backward_scratch_floats(int64_t m);

// Tensor-core GEMMs of the backward (gemm_umma.cu): split-bf16 three-pass wgmma kernels for the wide layer shapes.  A kernel that
// gives up on a barrier writes its code (6xx) to `status`, the error word of the network being differentiated.
bool gemm_tn_tc_supported(int N, int K);
// mask_bits: 1-bit ReLU mask of the output, [16 groups][M] uint16 (one plane of ActPlanes::bits), or NULL.  wimage: the packed W.
int launch_gemm_nn_tc(const float* A, int lda, const float* W, int ldw, float* C, int ldc, int64_t M, int N, int accumulate,
                      const uint16_t* mask_bits, DeviceBuffer& wimage, int32_t* status, cudaStream_t st);
// One product of a batched dW launch (gemm_umma.cu): C[N, K] += A[M, N]^T B[M, K]; b_cm != 0: B is column-major with that column
// stride; transpose: A is the wide operand and the result goes to C[K, N].
constexpr int TN_MAX_BATCH = 8;
struct TnProblem {
  const float* A; const float* B; float* C; float* colsum;
  int64_t b_cm;
  int lda, ldb, ldc, K, transpose;
};
// partial: the per-CTA partial products, reduced in a fixed order.
int launch_gemm_tn_tc_batch(const TnProblem* probs, int n, int64_t M, int N, DeviceBuffer& partial, int32_t* status, cudaStream_t st);

// Emptiness regulariser (penalizer.cu)
int launch_penalizer_forward(const float* raw, const float* z, const float* depth, const float* rays_d, int64_t n, int s, int c,
                             float tol, float w, void* partials, float* loss, cudaStream_t st);
int launch_penalizer_backward(const float* raw, const float* z, const float* depth, const float* rays_d, int64_t n, int s, int c,
                              float tol, float w, const void* state, const float* g_loss, float* d_raw, int accumulate,
                              cudaStream_t st);
size_t penalizer_state_bytes();
size_t penalizer_partials_bytes(int64_t n, int s, int c);
int launch_penalizer_merge(const void* states, int world, int c, void* state, float* loss, cudaStream_t st);

// Hungarian-matched instance loss (evaluator.cu)
int launch_hungarian_costs(const float* pred, const int32_t* gt_row, int64_t n, int k, float* cost_ce, float* cost_siou,
                           float* tp, float* s_sum, float* cnt, cudaStream_t st);
int launch_ins_loss_grad(const float* pred, const int32_t* gt_row, int64_t n, int64_t n_norm, int k, const int32_t* row_of_col,
                         const int32_t* n_valid, const float* tp, const float* s_sum, const float* cnt, const float* g3, float* d_pred,
                         cudaStream_t st);
int launch_label_rows(const int32_t* labels, int64_t n, int k, int32_t* gt_row, int32_t* n_valid, cudaStream_t st);
int launch_hungarian_assign(const float* cost_ce, const float* cost_siou, const float* s_sum, const int32_t* n_valid, int64_t n, int k,
                            int32_t* row_of_col, float* loss3, cudaStream_t st);
int ins_status_take();
int launch_label_bitmap(const int32_t* labels, int64_t n, uint32_t* bitmap, cudaStream_t st);
int launch_label_rows_merged(const uint32_t* bitmaps, int world, const int32_t* labels, int64_t n, int k, int32_t* gt_row,
                             int32_t* n_valid, cudaStream_t st);
int launch_hungarian_partials(const float* pred, const int32_t* gt_row, int64_t n, int k, double* partials, cudaStream_t st);
int launch_hungarian_costs_merged(const double* partials, int world, int64_t n, int k, float* cost_ce, float* cost_siou, float* tp,
                                  float* s_sum, float* cnt, cudaStream_t st);

// Mesh extraction (mesh.cu).  Transforms are row-major 4x4 float64 host arrays, extents 3 float64 host values.
// Per-context device buffers of the mesh entry points (the marching-cubes scans and the cleanup's compaction share some), and
// what the last marching-cubes count pass classified: mc_emit must see the same grid.
struct MeshState {
  DeviceBuffer eflags, cases, vcnt, vscan, tcnt, tscan, temp, totals, keys_in, keys_out, vals_in, vals_out, parent, size;
  DeviceBuffer edit_t, edit_flag, edit_pos;   // the edited sweep's slab: target points, in-box flags and their scan
  const float* grid = nullptr;
  int nx = 0, ny = 0, nz = 0;
  float level = 0.f;
  int64_t nv = -1, nt = -1;
};
int launch_grid_points(const double* T16, const double* ext3, int dim, int64_t begin, int64_t count, float* pts, cudaStream_t st);
int launch_occupancy(const float* raw, int64_t n, int c, float voxel, float* occ, cudaStream_t st);
// the same with an object selection: occ = 0 where the point's label is not kept; labels [n] int16 (may be NULL)
int launch_occupancy_objects(const float* raw, int64_t n, int c, float voxel, const ObjMask& keep, float* occ, int16_t* labels,
                             cudaStream_t st);
int mc_count(MeshState& s, const float* grid, int nx, int ny, int nz, float level, int64_t* counts, cudaStream_t st);
int mc_emit(MeshState& s, const float* grid, int nx, int ny, int nz, float level, float* verts, int32_t* tris, cudaStream_t st);
int launch_to_scene(const float* v, int64_t n, const double* T16, const double* ext3, int dim, float* out, cudaStream_t st);
int mesh_normals(MeshState& s, const float* v, int64_t nv, const int32_t* tris, int64_t nt, float* normals, cudaStream_t st);
int mesh_clusters(MeshState& s, const int32_t* tris, int64_t nt, int64_t nv, int32_t* cluster, int32_t* cluster_size, cudaStream_t st);
int mesh_clean(MeshState& s, const float* v, const float* nrm, int64_t nv, const int32_t* tris, int64_t nt, const int32_t* csize,
               int min_cluster, float* out_v, float* out_n, int32_t* out_t, int64_t* counts, cudaStream_t st);
int launch_label_rays(const float* v, const float* nrm, int64_t n, float near_z, float* ro, float* rd, cudaStream_t st);
int launch_argmax_rows(const float* x, int64_t n, int c, int64_t* out, cudaStream_t st);

// Meshing an edited scene (mesh.cu; DESIGN.md, "Meshing an edited scene").  One checked move of dmnerf_mesh_occupancy_edit: the
// 3x4 move and the grid's index map u = inv (t - b) in fp64, the box in index units, the piece (bits NULL: none).
struct EditMove {
  double trans[12];
  double inv[9];
  double b[3];
  double lo[3], hi[3];
  Region piece;
  int32_t label, rest_drop, empty;   // empty: the box holds no point, nothing is evaluated
};
// d -> m, checked against the grid (dim, transform, extents) and the bound network's ins_num
int edit_move_from_abi(const dmnerf_edit_move& d, const double* T16, const double* ext3, int dim, int ins_num, EditMove& m,
                       const char* who, int i);
// Points [begin, begin + count) of the grid: their targets under m, the boxed ones compacted in order into pts [*n_eval, 3];
// *n_eval read back (synchronises).
int edit_targets(MeshState& s, const double* T16, const double* ext3, int dim, const EditMove& m, int64_t begin, int64_t count,
                 float* pts, int64_t* n_eval, cudaStream_t st);
// take / vacate of m on the same points, raw [n_eval, c]: the network at the compacted targets of the last edit_targets
int edit_apply(MeshState& s, const double* T16, const double* ext3, int dim, const EditMove& m, int64_t begin, int64_t count,
               const float* raw, int c, float voxel, float level, float* occ, int16_t* labels, cudaStream_t st);
int launch_vertex_labels(const float* v, int64_t n, const float* occ, const int16_t* labels, int dim, float level, int16_t* out,
                         cudaStream_t st);
// The region of a move (bits NULL: none), checked: dim and map, the moved label among the labels it applies to (exchanger.cu).
int piece_region(const dmnerf_region& d, int mv, Region& r, const char* who, int i);

// Object inventory (inventory.cu): per-group integer statistics and fp64 spans of the solid points of a labelled grid.
// Per-context device buffers: everything a call reads back (status word first), and its inputs.
struct InventoryState {
  DeviceBuffer out, in;
};
int object_voxels(InventoryState& s, const float* occ, const int16_t* labels, int dim, float level, int n_labels,
                  const int32_t* boxes_host, int64_t* moments_host, uint32_t* hist_host, cudaStream_t st);
int object_spans(InventoryState& s, const float* occ, const int16_t* labels, int dim, float level, int n_labels,
                 const int32_t* boxes_host, const double* axes_host, double* spans_host, cudaStream_t st);

// Connected components (components.cu): the solid points of a labelled grid split into canonically numbered components.
// Per-context device buffers: the status words a call reads back, the chunk counts and the scan's storage.
struct ComponentsState {
  DeviceBuffer status, counts, temp;
};
int object_components(ComponentsState& s, const float* occ, const int16_t* labels, int dim, float level, int n_labels,
                      int connectivity, int32_t* comp, int64_t* n_components_host, cudaStream_t st);
int component_table(ComponentsState& s, const int32_t* comp, const int16_t* labels, int dim, int64_t n_comp, int16_t* label,
                    int64_t* voxels, int64_t* root, cudaStream_t st);
int component_groups(ComponentsState& s, const int32_t* comp, int dim, int64_t n_comp, const int16_t* lut, int discard,
                     int16_t* groups, cudaStream_t st);

// Region builders (region.cu).  Grids are [dim]^3 in C order; bits are region_words(dim) uint32 words, the tail zero.
int region_check(int dim, const float* map12, const char* who);      // dim in range, map finite (map12 may be NULL)
// The ABI region d as r, checked: bits not NULL, then region_check.
int region_from_abi(const dmnerf_region& d, Region& r, const char* who);
int region_pack(const int32_t* ids, int dim, const uint32_t* table, int64_t n_ids, uint32_t* bits, cudaStream_t st);
// tmp: region_words(dim) device words, needed when r >= 2
int region_dilate(const uint32_t* in, int dim, int r, int connectivity, int invert, uint32_t* out, uint32_t* tmp, cudaStream_t st);
int region_contains(const Region& r, const float* pts, int64_t n, uint8_t* out, cudaStream_t st);   // r from region_from_abi

// Test-view evaluation (metrics.cu)
int64_t eval_workspace_bytes(int64_t n, int k, int H, int W);
int eval_image(const float* rgb, const float* gt, int H, int W, void* ws, dmnerf_eval_result* res, cudaStream_t st);
int ins_eval(const float* ins, int64_t n, int k, const int32_t* gt_row, int gt_num, const float* mask, const int32_t* mask_labels,
             int mask_below, int64_t* pred_label, void* ws, dmnerf_eval_result* res, cudaStream_t st);
int calculate_ap(const float* iou, const float* conf, int m, int gt_number, float* ap6, cudaStream_t st);
int ins_dense_rows(const float* gt_ins, int64_t n, int k, int gt_num, int32_t* rows, cudaStream_t st);
int label_colors(const void* labels, int is64, int64_t n, const uint8_t* lut, int n_lut, uint8_t* out, cudaStream_t st);

}  // namespace dmnerf
