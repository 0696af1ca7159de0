/*
 * dmnerf_b200.h -- C ABI of the H100-native (sm_90a) DM-NeRF volumetric renderer (libdmnerf_b200.so).
 *
 * The reference (vLAR-group/DM-NeRF) has no FFI: its boundary is the Python call surface
 *   networks/render.py:31   dm_nerf(rays, pos_embedder, view_embedder, model_coarse, model_fine, z_vals_coarse, args)
 *   networks/render.py:6    render_train(raw, z_vals, rays_d)
 *   networks/dm_nerf.py:80  DM_NeRF.forward(x)
 *   networks/dm_nerf.py:37  Embedder.embed(x)
 *   networks/helpers.py:123 sample_pdf(bins, weights, N_samples, det)
 * Each entry point below names the reference function it replaces.  All pointers are plain device
 * pointers (float32, row-major, contiguous) unless the name ends in _host; `stream` is a cudaStream_t
 * passed as void* (NULL = legacy default stream).  Every function returns 0 on success and a non-zero
 * status otherwise (never throws); dmnerf_last_error() returns a thread-local message.  No torch types
 * cross this boundary -- see INTEGRATION.md for the ctypes binding the Python host layer uses.
 */
#ifndef DMNERF_B200_H_
#define DMNERF_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define DMNERF_API __attribute__((visibility("default")))
#else
#define DMNERF_API
#endif

#define DMNERF_ABI_VERSION 1
#define DMNERF_N_PARAMS 30          /* tensors in DM_NeRF.state_dict() order, networks/dm_nerf.py:65-78 */
#define DMNERF_CH_POS 63            /* get_embedder(10): 3 + 3*2*10, networks/dm_nerf.py:41-55 */
#define DMNERF_CH_DIR 27            /* get_embedder(4) */
#define DMNERF_MAX_INS 127          /* ins_num + 1 <= 128 */

/* MLP implementation selector */
#define DMNERF_IMPL_AUTO 0          /* tensor-core path when available for the shape, else SIMT */
#define DMNERF_IMPL_SIMT 1          /* fp32 CUDA-core reference kernel */
#define DMNERF_IMPL_UMMA 2          /* wgmma tensor-core kernel, bf16x3 split operands, fp32 accumulate */

/* dmnerf_render_* flags */
#define DMNERF_FLAG_PERTURB   1     /* args.perturb > 0: t_rand and u must be given (render.py:40-47, helpers.py:135) */
#define DMNERF_FLAG_WANT_RAW  2     /* materialise raw_coarse / raw_fine (training, penalizer.py) */
#define DMNERF_FLAG_KEEP_INS  4     /* keep all ins_num+1 instance channels, no detach: manipulator.py:86-105 */

typedef struct dmnerf_ctx dmnerf_ctx;

/* All per-ray inputs/outputs of one dm_nerf() call (networks/render.py:31-96).  Any output pointer
 * may be NULL (not written).  Shapes: N rays, S coarse samples, I importance samples, F = S + I,
 * C = 4 + ins_num + 1. */
typedef struct dmnerf_render_io {
  const float* rays_o;       /* [N,3] */
  const float* rays_d;       /* [N,3] un-normalised */
  const float* z_coarse;     /* [S] shared row (z_row_stride = 0) or [N,S] (z_row_stride = S) */
  int64_t      z_row_stride;
  const float* t_rand;       /* [N,S] stratified jitter uniforms or NULL (render.py:46) */
  const float* u;            /* [N,I] inverse-CDF uniforms or NULL => linspace(0,1,I) (helpers.py:131-135) */
  float* rgb_coarse;         /* [N,3] */
  float* rgb_fine;           /* [N,3] */
  float* depth_coarse;       /* [N] */
  float* depth_fine;         /* [N] */
  float* acc_coarse;         /* [N]  sum of weights (north_star acc_map) */
  float* acc_fine;           /* [N] */
  float* ins_coarse;         /* [N,ins_num] post-sigmoid, last class dropped (render.py:24-26) */
  float* ins_fine;           /* [N,ins_num] */
  float* z_vals_coarse;      /* [N,S] (after jitter) */
  float* z_vals_fine;        /* [N,F] sorted */
  float* weights_coarse;     /* [N,S] */
  float* weights_fine;       /* [N,F] */
  float* raw_coarse;         /* [N,S,C] only with DMNERF_FLAG_WANT_RAW */
  float* raw_fine;           /* [N,F,C] */
} dmnerf_render_io;

DMNERF_API int         dmnerf_abi_version(void);
DMNERF_API const char* dmnerf_last_error(void);

DMNERF_API int dmnerf_ctx_create(int device, dmnerf_ctx** out);
DMNERF_API int dmnerf_ctx_destroy(dmnerf_ctx* ctx);

/* Bind one network's LIVE parameter storage (30 device pointers, state_dict order) and re-pack the
 * tensor-core operand image.  net: 0 = coarse, 1 = fine.  Replaces model.load_state_dict()/the
 * nn.Module parameter reads of DM_NeRF.forward (networks/dm_nerf.py:80-106).  Call again after every
 * in-place optimizer update. */
DMNERF_API int dmnerf_set_weights(dmnerf_ctx* ctx, int net, const float* const* params, int n_params, int ins_num,
                       void* stream);

/* Embedder.embed, networks/dm_nerf.py:37-38: x [M,3] -> out [M, 3 + 6*n_freqs]. */
DMNERF_API int dmnerf_posenc(const float* x, int64_t m, int n_freqs, float* out, void* stream);

/* DM_NeRF.forward, networks/dm_nerf.py:80-106: x [M,90] -> out [M,C]. */
DMNERF_API int dmnerf_mlp_forward(dmnerf_ctx* ctx, int net, const float* x, int64_t m, float* out, int impl, void* stream);

/* Same network evaluated at points given as rays + depths (render.py:49-61 fused: pts = o + d z,
 * both embeddings, MLP).  z [N,S] -> out [N,S,C]. */
DMNERF_API int dmnerf_mlp_forward_rays(dmnerf_ctx* ctx, int net, const float* rays_o, const float* rays_d, const float* z,
                            int64_t n, int s, float* out, int impl, void* stream);

/* render_train, networks/render.py:6-28 (keep_all_ins != 0: manipulator_render, manipulator.py:86-105).
 * raw [N,S,C], z [N,S], rays_d [N,3] -> rgb [N,3], weights [N,S], depth [N], ins [N, C-5 or C-4], acc [N]. */
DMNERF_API int dmnerf_composite(const float* raw, const float* z, const float* rays_d, int64_t n, int s, int c,
                     int keep_all_ins, float* rgb, float* weights, float* depth, float* ins, float* acc,
                     void* stream);

/* sample_pdf, networks/helpers.py:123-155.  bins [N,nb], weights [N,nb-1]; u [N,ns] or NULL (det). */
DMNERF_API int dmnerf_sample_pdf(const float* bins, const float* weights, int64_t n, int n_bins, int n_samples,
                      const float* u, float* out, void* stream);

/* torch.sort(torch.cat([a, b], -1), -1).values, networks/render.py:70.  a [N,na], b [N,nb] -> [N,na+nb]. */
DMNERF_API int dmnerf_sort_concat(const float* a, const float* b, int64_t n, int na, int nb, float* out, void* stream);

/* get_rays_k, networks/helpers.py:50-61: K (HOST, row-major 3x3) and c2w (HOST, row-major, at least its top 3x4 = 12 floats)
 * -> rays_o, rays_d [H*W, 3] on the device, pixel-major like the reference's reshape(-1, 3). */
DMNERF_API int dmnerf_get_rays(const float* K_host, const float* c2w_host, int H, int W, float* rays_o, float* rays_d, void* stream);

/* The rays of selected pixels only -- the training-side ray selection get_select_full / get_select_crop,
 * networks/helpers.py:64-111, builds all H*W rays per iteration to keep 1024-3072 of them: pixels [n] (DEVICE, int64,
 * row * W + column) -> rays_o, rays_d [n,3], bit-identical to the rows get_rays_k would produce. */
DMNERF_API int dmnerf_get_rays_at(const float* K_host, const float* c2w_host, int H, int W, const int64_t* pixels, int64_t n,
                                  float* rays_o, float* rays_d, void* stream);
/* The same with the pose in DEVICE memory (3 rows of 4 floats, c2w_row_stride floats apart): train_dmsr.py:27 hands
 * get_select_full a CUDA tensor, and reading it back would synchronise every iteration. */
DMNERF_API int dmnerf_get_rays_at_dev(const float* K_host, const float* c2w_dev, int64_t c2w_row_stride, int H, int W,
                                      const int64_t* pixels, int64_t n, float* rays_o, float* rays_d, void* stream);
/* n distinct pseudo-random pixels (row * W + column, DEVICE int64) of an H x W image from a keyed bijection of [0, H*W): the
 * opt-in device-side replacement of np.random.choice(H*W, N, replace=False) in helpers.py:100 (uniform without replacement, but
 * NOT numpy's random stream). */
DMNERF_API int dmnerf_select_pixels(uint64_t seed, int H, int W, int64_t n, int64_t* pixels, void* stream);

/* Hungarian-matched instance loss, networks/evaluator.py:19-74 (ins_criterion / hungarian; train_dmsr.py:38-45).
 * dmnerf_hungarian_costs: pred [N,ins_num] (rendered instance probabilities), gt_row [N] (int32: index of the ray's label among
 * the sorted distinct labels of the batch, evaluator.py:21-25) -> cost_ce, cost_siou [ins_num,ins_num] (row = ground-truth
 * object, column = prediction channel; evaluator.py:60-67) plus the sums the backward needs: tp [ins_num,ins_num],
 * col_sum [ins_num] (sum_n pred), row_count [ins_num].  The assignment (scipy linear_sum_assignment, evaluator.py:45-47) runs on
 * the host on the [valid x ins_num] corner of cost_ce + cost_siou, as in the reference.
 * dmnerf_ins_loss_backward: d_pred [N,ins_num] = g[0] d valid_ce + g[1] d invalid_ce + g[2] d valid_siou (evaluator.py:27-36);
 * row_of_col [ins_num] (DEVICE int32) = matched ground-truth row of every prediction channel or -1; g_losses = 3 DEVICE floats. */
DMNERF_API int dmnerf_hungarian_costs(const float* pred, const int32_t* gt_row, int64_t n, int ins_num, float* cost_ce,
                                      float* cost_siou, float* tp, float* col_sum, float* row_count, void* stream);
DMNERF_API int dmnerf_ins_loss_backward(const float* pred, const int32_t* gt_row, int64_t n, int ins_num,
                                        const int32_t* row_of_col, int n_valid, const float* tp, const float* col_sum,
                                        const float* row_count, const float* g_losses, float* d_pred, void* stream);

/* The same loss with the assignment ON THE DEVICE: no device->host hop in the training iteration (the reference's
 * valid_scores.cpu() + scipy call, evaluator.py:43-45, is its last synchronisation point).
 * dmnerf_ins_label_rows: labels [N] (int32 object ids in [0, 65536)) -> gt_row [N] = rank of the ray's label among the distinct
 *   labels of the batch (torch.unique order, evaluator.py:21-25) and n_valid[0] = their number (DEVICE int32; -1 when a label is
 *   out of range or there are more distinct labels than ins_num).
 * dmnerf_hungarian_assign: scipy.optimize.linear_sum_assignment's algorithm (shortest augmenting paths, fp64 duals, scipy's tie
 *   rule) on rows 0..n_valid-1 of cost_ce + cost_siou -> row_of_col [ins_num] (matched row or -1) and
 *   losses[3] = { valid_ce, invalid_ce, valid_siou } (evaluator.py:27-36; NaN after rejected labels).
 * dmnerf_ins_loss_backward_dev: dmnerf_ins_loss_backward with n_valid read from the device (zero gradient after rejected labels).
 * dmnerf_ins_status_take: returns and clears the error word of rejected labels (0 = none; mapped host memory, no synchronisation). */
DMNERF_API int dmnerf_ins_label_rows(const int32_t* labels, int64_t n, int ins_num, int32_t* gt_row, int32_t* n_valid, void* stream);
DMNERF_API int dmnerf_hungarian_assign(const float* cost_ce, const float* cost_siou, const float* col_sum, const int32_t* n_valid,
                                       int64_t n, int ins_num, int32_t* row_of_col, float* losses, void* stream);
DMNERF_API int dmnerf_ins_loss_backward_dev(const float* pred, const int32_t* gt_row, int64_t n, int ins_num,
                                            const int32_t* row_of_col, const int32_t* n_valid, const float* tp, const float* col_sum,
                                            const float* row_count, const float* g_losses, float* d_pred, void* stream);
DMNERF_API int dmnerf_ins_status_take(void);

/* Coarse depths, networks/render.py:40-47: z_out[n, i] = z_in row (shared when z_row_stride = 0), jittered inside its
 * stratum by t_rand [N,S] when given. */
DMNERF_API int dmnerf_stratify(const float* z_in, int64_t z_row_stride, const float* t_rand, int64_t n, int s, float* z_out,
                    void* stream);

/* networks/render.py:66-70 in one launch: z_mid, sample_pdf on weights[1:-1] (u [N,I] or NULL = deterministic), concat with
 * the coarse depths and sort.  z_c [N,S], w_c [N,S] -> z_fine [N,S+I]. */
DMNERF_API int dmnerf_hier_sample(const float* z_c, const float* w_c, const float* u, int64_t n, int s, int n_importance,
                       float* z_fine, void* stream);

/* ---- training (BASELINE config 4; reference train_dmsr.py:62-64 total_loss.backward()) -------------------------------
 * The training forward evaluates the network in exact fp32 and keeps the activations the backward needs:
 * dmnerf_act_floats_per_sample() floats per sample in `acts` (device buffer owned by the caller). */
DMNERF_API int dmnerf_act_floats_per_sample(void);
DMNERF_API int64_t dmnerf_mlp_backward_scratch_floats(int64_t m);

/* DM_NeRF.forward with saved activations.  Pass either x [M,90] (rays_* NULL) or rays_o/rays_d [N,3] + z [N,S] (x NULL,
 * m = N*S).  out [M,C].  impl: DMNERF_IMPL_SIMT = exact fp32; DMNERF_IMPL_UMMA / AUTO = the tensor-core kernel, whose folded heads
 * do not produce the rgb_feature / ins_feature planes -- pass feats_missing = 1 to dmnerf_mlp_backward in that case.  Both
 * kernels also keep the ReLU masks (1 bit per unit) the fused gradient chain of the backward reads. */
DMNERF_API int dmnerf_mlp_forward_train(dmnerf_ctx* ctx, int net, const float* x, const float* rays_o, const float* rays_d,
                             const float* z, int64_t m, int s, float* out, float* acts, int impl, void* stream);

/* Gradient of a scalar loss w.r.t. the 30 parameters of network `net` given d_out = dL/d(out) [M,C] and the activations
 * saved by dmnerf_mlp_forward_train.  grads: 30 device buffers (state_dict order, parameter shapes), overwritten.
 * Gradient routing follows the reference (networks/dm_nerf.py:95: the instance branch reads h.detach()).
 * scratch: dmnerf_mlp_backward_scratch_floats(m) floats.  feats_missing is a flag word: bit 0 = the forward did not write the
 * feature planes (tensor-core forward), bit 1 = the caller has already zero-filled `grads` (one fill instead of 30 memsets).
 * M >= 512: the heads are folded like in the forward, one masked split-bf16 wgmma GEMM per layer carries the gradient
 * through the trunk and batched wgmma GEMMs form the weight gradients; smaller batches and DMNERF_BWD_IMPL=simt use fp32
 * CUDA-core kernels. */
DMNERF_API int dmnerf_mlp_backward(dmnerf_ctx* ctx, int net, float* acts, const float* d_out, int64_t m, float* const* grads,
                        float* scratch, int feats_missing, void* stream);

/* Backward of render_train (networks/render.py:6-28): upstream gradients of rgb_map [N,3], depth_map [N], acc_map [N],
 * ins_map [N, C-5 | C-4] and weights [N,S] (any may be NULL) -> d_raw [N,S,C] (added to d_raw when accumulate != 0).
 * The instance map sees detached weights unless keep_all_ins (render.py:22-23 vs manipulator.py:100). */
DMNERF_API int dmnerf_composite_backward(const float* raw, const float* z, const float* rays_d, int64_t n, int s, int c,
                              int keep_all_ins, const float* g_rgb, const float* g_depth, const float* g_acc,
                              const float* g_ins, const float* g_weights, float* d_raw, int accumulate, void* stream);

/* Frame driver: the test-time loop of render_test (networks/tester.py:55-76) for one camera, without the ray upload: rays
 * are generated on the device from K / c2w (get_rays_k, helpers.py:50-61), the shared coarse depth row from near / far
 * (z_val_sample, helpers.py:114-119), and pixels [ray_begin, ray_begin + ray_count) of the H x W frame (pixel-major, the
 * reference's reshape(-1, 3)) are rendered by dm_nerf(); every non-NULL OUTPUT field of `out_host` (host memory, ray_count
 * rows) is filled; its input fields are ignored.  Deterministic path only (perturb = 0).  Synchronises the stream. */
DMNERF_API int dmnerf_render_frame_host(dmnerf_ctx* ctx, const float* K_host, const float* c2w_host, int H, int W, float near_z,
                                        float far_z, int64_t ray_begin, int64_t ray_count, int n_coarse, int n_importance,
                                        int flags, int impl, const dmnerf_render_io* out_host, void* stream);

/* Point query: the network at m points with explicit view directions, both embedded inside the kernel
 * (pts [m,3], viewdirs [m,3] used as they are -- no normalisation) -> out [m, 4+ins_num+1].  This is the grid sweep of
 * tools/mesh_generator.py:36-49 (256^3 points, zero view directions) without the [m,90] embedded tensor in HBM. */
DMNERF_API int dmnerf_mlp_forward_points(dmnerf_ctx* ctx, int net, const float* pts, const float* viewdirs, int64_t m, float* out,
                                         int impl, void* stream);

/* exchanger, networks/manipulator.py:18-83: per-sample swap of network outputs between the original rays and up to 8
 * transformed ("target") ray sets of an object edit.  ori_raw [N,S,C] is edited IN PLACE; tar_raws / tar_accs are HOST arrays
 * of n_moves DEVICE pointers ([N,S,C] / [N,C-4]); ori_acc [N,C-4] and tar_accs are the rendered instance maps with every
 * channel kept (manipulator_render); move_labels is a HOST array.  Outputs: int64 per-sample labels of the original and of the
 * last target after the occlusion fixes. */
DMNERF_API int dmnerf_exchanger(float* ori_raw, const float* const* tar_raws, const float* ori_acc, const float* const* tar_accs,
                                const int* move_labels, int n_moves, int64_t n, int s, int c, int64_t* ori_label,
                                int64_t* tar_label, void* stream);

/* "Emptiness" regulariser on the per-sample object logits: emptiness_penalizer / ins_penalizer, networks/penalizer.py:5-62
 * (train_dmsr.py:53-60).  raw [N,S,C], z_vals [N,S], depth [N] (the rendered depth map, treated as a constant),
 * rays_d [N,3] -> loss[1] (device).  `state` is caller-provided device scratch of dmnerf_penalizer_state_bytes() bytes that
 * carries the mask populations from the forward to the backward call.  Backward (g_loss is a DEVICE scalar): accumulate == 0
 * writes d_raw = g_loss[0] * dL/draw for EVERY channel (zeros in channels 0..3: no zero-fill needed); accumulate != 0 adds the
 * gradient to channels 4.. and leaves channels 0..3 untouched. */
DMNERF_API int64_t dmnerf_penalizer_state_bytes(void);
DMNERF_API int dmnerf_penalizer_forward(const float* raw, const float* z_vals, const float* depth, const float* rays_d, int64_t n,
                                        int s, int c, float tolerance, float deta_w, void* state, float* loss, void* stream);
DMNERF_API int dmnerf_penalizer_backward(const float* raw, const float* z_vals, const float* depth, const float* rays_d, int64_t n,
                                         int s, int c, float tolerance, float deta_w, const void* state, const float* g_loss,
                                         float* d_raw, int accumulate, void* stream);

/* dm_nerf(), networks/render.py:31-96, whole per-ray pipeline on device buffers. */
DMNERF_API int dmnerf_render_forward(dmnerf_ctx* ctx, const dmnerf_render_io* io, int64_t n_rays, int n_coarse,
                          int n_importance, int flags, int impl, void* stream);

/* Same call with HOST buffers (pageable or pinned): copies rays in, renders, copies every non-NULL
 * output back, and synchronises the stream.  This is the end-to-end entry point bench.py times.
 * A batch of >= 131 072 rays is rendered in four parts (same bits: rays are independent) whose uploads / downloads travel on a
 * second stream while the neighbouring parts are rendered: only the first upload and the last download are exposed. */
DMNERF_API int dmnerf_render_forward_host(dmnerf_ctx* ctx, const dmnerf_render_io* io_host, int64_t n_rays, int n_coarse,
                               int n_importance, int flags, int impl, void* stream);

/* Synchronise `stream` and report any asynchronous failure of the kernels launched through `ctx` (CUDA errors and
 * the tensor-core kernel's bounded-wait protocol check). */
DMNERF_API int dmnerf_sync_check(dmnerf_ctx* ctx, void* stream);

/* Per-stage device timing of dmnerf_render_forward (CUDA events recorded on the launch stream around each stage):
 * enable != 0 switches recording on.  dmnerf_profile_read synchronises the last recorded events and writes the
 * elapsed milliseconds of the last render call: [0] coarse depths, [1] coarse network, [2] coarse composite,
 * [3] importance sampling + merge, [4] fine network, [5] fine composite.  n_out must be >= 6. */
#define DMNERF_N_STAGES 6
DMNERF_API int dmnerf_profile_enable(dmnerf_ctx* ctx, int enable);
DMNERF_API int dmnerf_profile_read(dmnerf_ctx* ctx, float* ms_out, int n_out);

/* ---- mesh extraction: mesh_main, tools/mesh_generator.py (+ tools/visualizer.py) ----------------------------------------
 * transform_host: row-major 4x4 float64 (scene_transform = inv(to_origin), :23-25); extents_host: 3 float64 ([1.9, 7, 7], :26).
 * Conventions (vertex position, numbering, face-ambiguity rule, winding): DESIGN.md, "Mesh extraction".
 *
 * dmnerf_mesh_grid_points: points [begin, begin + count) of the dim^3 query grid (C order of the grid index), in the network's
 *   frame: make_3D_grid / grid_within_bound in float32 + the axis swap and flip of :28-29.  pts [count,3].
 * dmnerf_mesh_occupancy: the occupancy sweep (:33-63): network `net` at every grid point with zero view directions, slab points
 *   at a time (slab <= 0: 2^20), each slab reduced to occ = 1 - exp(-relu(sigma) * voxel) -> occ [dim,dim,dim].
 * dmnerf_mesh_mc_count / _mc_emit: marching cubes (:68-69) on any grid [nx,ny,nz] (DEVICE, C order), inside = value > level.
 *   count classifies, scans and reads back counts_host[0] = vertices, [1] = triangles (the one device->host read; fails on a grid
 *   holding NaN); emit (same grid and level) writes verts [V,3] in index units and tris [T,3] int32.
 * dmnerf_mesh_to_scene: index-space vertices -> scene space (:70-86): v / (dim - 1) in float32, then (q - 0.5) * 2 * extents / 2
 *   and the transform in float64, rounded to float32.
 * dmnerf_mesh_normals: area-weighted vertex normals (open3d compute_vertex_normals, visualizer.py:164), deterministic.
 * dmnerf_mesh_clusters: edge-connected triangle clusters (cluster_connected_triangles, visualizer.py:174): cluster [T] = smallest
 *   triangle index of the cluster, cluster_size [T] = its triangle count.
 * dmnerf_mesh_clean: clean_mesh (visualizer.py:169-194): triangles with cluster_size < min_cluster removed, then unreferenced
 *   vertices; order kept.  Outputs need room for nv / nt rows; counts_host[0..1] = kept vertices / triangles.  normals and
 *   out_normals may both be NULL.
 * dmnerf_mesh_label_rays: the per-vertex label rays (:106-113): rays_d = -normal, rays_o = v - rays_d * 0.03 * near, both in the
 *   network's frame.
 * dmnerf_argmax_rows: torch.argmax(x, -1) of x [n,c] -> int64 [n] (first maximum; NaN counts as the maximum). */
DMNERF_API int dmnerf_mesh_grid_points(const double* transform_host, const double* extents_host, int dim, int64_t begin, int64_t count,
                                       float* pts, void* stream);
DMNERF_API int dmnerf_mesh_occupancy(dmnerf_ctx* ctx, int net, const double* transform_host, const double* extents_host, int dim,
                                     float voxel, int64_t slab, float* occ, void* stream);
DMNERF_API int dmnerf_mesh_mc_count(dmnerf_ctx* ctx, const float* grid, int nx, int ny, int nz, float level, int64_t* counts_host,
                                    void* stream);
DMNERF_API int dmnerf_mesh_mc_emit(dmnerf_ctx* ctx, const float* grid, int nx, int ny, int nz, float level, float* verts, int32_t* tris,
                                   void* stream);
DMNERF_API int dmnerf_mesh_to_scene(const float* verts, int64_t n, const double* transform_host, const double* extents_host, int dim,
                                    float* out, void* stream);
DMNERF_API int dmnerf_mesh_normals(dmnerf_ctx* ctx, const float* verts, int64_t nv, const int32_t* tris, int64_t nt, float* normals,
                                   void* stream);
DMNERF_API int dmnerf_mesh_clusters(dmnerf_ctx* ctx, const int32_t* tris, int64_t nt, int64_t nv, int32_t* cluster, int32_t* cluster_size,
                                    void* stream);
DMNERF_API int dmnerf_mesh_clean(dmnerf_ctx* ctx, const float* verts, const float* normals, int64_t nv, const int32_t* tris, int64_t nt,
                                 const int32_t* cluster_size, int min_cluster, float* out_verts, float* out_normals, int32_t* out_tris,
                                 int64_t* counts_host, void* stream);
DMNERF_API int dmnerf_mesh_label_rays(const float* verts, const float* normals, int64_t n, float near_z, float* rays_o, float* rays_d,
                                      void* stream);
DMNERF_API int dmnerf_argmax_rows(const float* x, int64_t n, int c, int64_t* out, void* stream);

/* Number of kernels this library has launched on the calling thread's contexts since load. */
DMNERF_API int64_t dmnerf_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* DMNERF_B200_H_ */
