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

#define DMNERF_ABI_VERSION 4
#define DMNERF_N_PARAMS 30          /* tensors in DM_NeRF.state_dict() order, networks/dm_nerf.py:65-78 */
#define DMNERF_CH_POS 63            /* get_embedder(10): 3 + 3*2*10, networks/dm_nerf.py:41-55 */
#define DMNERF_CH_DIR 27            /* get_embedder(4) */
#define DMNERF_MAX_INS 127          /* ins_num + 1 <= 128 */

/* MLP implementation selector */
#define DMNERF_IMPL_AUTO 0          /* DMNERF_IMPL_UMMA: a bound network always has its tensor-core image */
#define DMNERF_IMPL_SIMT 1          /* fp32 CUDA-core reference kernel */
#define DMNERF_IMPL_UMMA 2          /* wgmma tensor-core kernel, bf16x3 split operands, fp32 accumulate */
/* Preview precision, INFERENCE ONLY: the same tensor-core network run once with fp16 operands and fp32 accumulation (1/3 of
 * the MMAs, 1/2 of the weight bytes).  Accepted by dmnerf_mlp_forward(_rays/_points), dmnerf_render_forward(_host) and
 * dmnerf_render_frame_host (with DMNERF_FLAG_WANT_RAW the stage kernels run it too).  Its weight image is packed
 * on the first fp16 call after each dmnerf_set_weights, from the bound weights as they are then and the folded heads and
 * biases packed by that dmnerf_set_weights: as for the exact image, weights changed in place take effect only through a new
 * dmnerf_set_weights.  Measured against fp64 (DESIGN.md section 10, H100): network outputs rel. L2 2.8e-4 - 4.6e-4,
 * rendered rgb 54 - 62 dB PSNR on typical rays, argmax labels >= 0.99 agreement.  fp16 stops at 65504: a weight above it fails
 * the call at pack time, and a stored activation above it fails the call after the kernel (these fp16 calls synchronise
 * the stream to deliver that verdict) -- render such a network with DMNERF_IMPL_UMMA.  dmnerf_mlp_forward_train rejects it
 * (training and every backward stay exact), and dmnerf_mesh_occupancy, which has no impl, stays exact on purpose:
 * its threshold decides the surface. */
#define DMNERF_IMPL_UMMA_F16 3

/* dmnerf_render_* flags */
#define DMNERF_FLAG_PERTURB   1     /* args.perturb > 0: t_rand and u must be given (render.py:40-47, helpers.py:135) */
#define DMNERF_FLAG_WANT_RAW  2     /* materialise raw_coarse / raw_fine (training, penalizer.py) */
#define DMNERF_FLAG_KEEP_INS  4     /* keep all ins_num+1 instance channels, no detach: manipulator.py:86-105 */
/* The render entry points reject any other flag bit. */

typedef struct dmnerf_ctx dmnerf_ctx;

/* A region (see "region selection" below). */
typedef struct dmnerf_region {
  const uint32_t* bits;      /* DEVICE, ceil(dim^3 / 32) words; the caller keeps them alive for the call */
  int32_t dim;
  int32_t outside_keep;      /* 1: a sample outside the grid is kept (in the piece); 0: dropped */
  float voxel_map[12];       /* row-major 3x4 [M | c]: network frame -> grid index */
  uint32_t applies[4];       /* labels the region applies to, bit k of word k / 32 */
} dmnerf_region;

/* The scene edit of one render call (see "object selection", "region selection" and "object appearance" below).  An edit
 * whose three members are all NULL is no edit. */
typedef struct dmnerf_edit {
  const uint32_t* keep;            /* HOST, 4 words of kept labels (bit k of word k / 32); NULL: every label */
  const dmnerf_region* region;     /* HOST struct; NULL: no region */
  const float* appearance;         /* HOST [appearance_labels][16]; NULL: no appearance */
  int32_t appearance_labels;
} dmnerf_edit;

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
  const dmnerf_edit* edit;   /* HOST: the scene edit, or NULL for none */
} dmnerf_render_io;

DMNERF_API int         dmnerf_abi_version(void);
DMNERF_API const char* dmnerf_last_error(void);

DMNERF_API int dmnerf_ctx_create(int device, dmnerf_ctx** out);
DMNERF_API int dmnerf_ctx_destroy(dmnerf_ctx* ctx);

/* Bind one network's LIVE parameter storage (30 device pointers, state_dict order) and re-pack the
 * tensor-core operand image.  net: 0 = coarse, 1 = fine.  Replaces model.load_state_dict()/the
 * nn.Module parameter reads of DM_NeRF.forward (networks/dm_nerf.py:80-106).  Call again after every
 * in-place optimizer update.  A call whose arguments are rejected (ctx, net, n_params, ins_num or a NULL
 * pointer) leaves the slot exactly as it was.  Otherwise the slot is bound only if the pack succeeds: after a
 * failed pack it is unbound, and every call that runs it fails until a dmnerf_set_weights succeeds. */
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
 * raw [N,S,C], z [N,S], rays_d [N,3] -> rgb [N,3], weights [N,S], depth [N], ins [N, C-5 or C-4], acc [N].
 * keep_host: an object selection over labels 0 .. C-5 (see "object selection" below), or NULL. */
DMNERF_API int dmnerf_composite(const float* raw, const float* z, const float* rays_d, int64_t n, int s, int c,
                     int keep_all_ins, const uint32_t* keep_host, float* rgb, float* weights, float* depth, float* ins,
                     float* acc, void* stream);

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

/* Hungarian-matched instance loss, networks/evaluator.py:19-74 (ins_criterion / hungarian; train_dmsr.py:38-45).  Every sum runs
 * in an order fixed by the sizes alone (no floating-point atomics), so the losses and gradients are reproducible bit for bit.
 * dmnerf_hungarian_costs: pred [N,ins_num] (rendered instance probabilities), gt_row [N] (int32: index of the ray's label among
 *   the sorted distinct labels of the batch, evaluator.py:21-25) -> cost_ce, cost_siou [ins_num,ins_num] (row = ground-truth
 *   object, column = prediction channel; evaluator.py:60-67) plus the sums the backward needs: tp [ins_num,ins_num],
 *   col_sum [ins_num] (sum_n pred), row_count [ins_num].  The assignment (scipy linear_sum_assignment, evaluator.py:45-47) runs
 *   either on the host on the [valid x ins_num] corner of cost_ce + cost_siou, as in the reference, or on the device:
 * dmnerf_ins_label_rows: labels [N] (int32 object ids in [0, 65536)) -> gt_row [N] = rank of the ray's label among the distinct
 *   labels of the batch (torch.unique order, evaluator.py:21-25) and n_valid[0] = their number (DEVICE int32; -1 when a label is
 *   out of range or there are more distinct labels than ins_num).
 * dmnerf_hungarian_assign: scipy.optimize.linear_sum_assignment's algorithm (shortest augmenting paths, fp64 duals, scipy's tie
 *   rule) on rows 0..n_valid-1 of cost_ce + cost_siou -> row_of_col [ins_num] (matched row or -1) and
 *   losses[3] = { valid_ce, invalid_ce, valid_siou } (evaluator.py:27-36; NaN after rejected labels).  With these two the
 *   training iteration has no device->host hop (the reference's valid_scores.cpu() + scipy call, evaluator.py:43-45, is its
 *   last synchronisation point).
 * dmnerf_ins_loss_backward: d_pred [n,ins_num] = g[0] d valid_ce + g[1] d invalid_ce + g[2] d valid_siou (evaluator.py:27-36)
 *   for n rows of a batch of n_global rays (n = n_global in one process); row_of_col [ins_num] (DEVICE int32) = matched
 *   ground-truth row of every prediction channel or -1; n_valid[0] (DEVICE int32) = the number of distinct labels (zero gradient
 *   when it is below 1: rejected labels); g_losses = 3 DEVICE floats.
 * dmnerf_ins_status_take: returns and clears the error word of rejected labels (0 = none; mapped host memory, no synchronisation). */
DMNERF_API int dmnerf_hungarian_costs(const float* pred, const int32_t* gt_row, int64_t n, int ins_num, float* cost_ce,
                                      float* cost_siou, float* tp, float* col_sum, float* row_count, void* stream);
DMNERF_API int dmnerf_ins_label_rows(const int32_t* labels, int64_t n, int ins_num, int32_t* gt_row, int32_t* n_valid, void* stream);
DMNERF_API int dmnerf_hungarian_assign(const float* cost_ce, const float* cost_siou, const float* col_sum, const int32_t* n_valid,
                                       int64_t n, int ins_num, int32_t* row_of_col, float* losses, void* stream);
DMNERF_API int dmnerf_ins_loss_backward(const float* pred, const int32_t* gt_row, int64_t n, int64_t n_global, int ins_num,
                                        const int32_t* row_of_col, const int32_t* n_valid, const float* tp, const float* col_sum,
                                        const float* row_count, const float* g_losses, float* d_pred, void* stream);
DMNERF_API int dmnerf_ins_status_take(void);

/* The same loss over a batch split into W contiguous shards (one per process, dmnerf_b200.distributed): each shard computes
 * partials, the caller all-gathers them, and every shard merges the W buffers in shard order, so every shard feeds bit-identical
 * inputs to dmnerf_hungarian_assign (which is passed the global N) and then calls dmnerf_ins_loss_backward for its own rows.
 * dmnerf_hungarian_costs is the one-shard case: it equals dmnerf_hungarian_partials followed by dmnerf_hungarian_costs_merged
 * with world = 1 bit for bit.
 * dmnerf_ins_label_bitmap: labels [n] -> bitmap [DMNERF_LABEL_WORDS] (DEVICE uint32): words 0..2047 mark the label values
 *   [0, 65536) present in the shard, word 2048 is 1 when a label is out of range (also posted to the status word: 701).
 * dmnerf_ins_label_rows_merged: bitmaps [world, DMNERF_LABEL_WORDS] (the gathered bitmaps, rank order) and the shard's labels [n]
 *   -> gt_row [n] = rank of the label among the distinct labels of the whole batch, n_valid[0] (dmnerf_ins_label_rows' rules:
 *   -1 and status 701 / 702 for an out-of-range label in any shard or more distinct labels than ins_num).
 * dmnerf_hungarian_partials: pred [n,ins_num], gt_row [n] -> partials [3 ins_num (ins_num + 1)] (DEVICE fp64), laid out
 *   A[k] | S[k] | B[k,k] | C[k,k] | TP[k,k] | cnt[k] with k = ins_num, element (g, p) at g * k + p:
 *   A[p] = sum log(1 - pred[:,p] + 1e-8), S[p] = sum pred[:,p], and over the rays of row g: B = sum log(pred + 1e-8),
 *   C = sum log(1 - pred + 1e-8), TP = sum pred, cnt = ray count.
 * dmnerf_hungarian_costs_merged: partials [world, 3 k (k + 1)] added in shard order -> cost_ce, cost_siou, tp, col_sum, row_count
 *   exactly as dmnerf_hungarian_costs computes them from those sums, normalised by n_global. */
#define DMNERF_LABEL_WORDS 2049
DMNERF_API int dmnerf_ins_label_bitmap(const int32_t* labels, int64_t n, uint32_t* bitmap, void* stream);
DMNERF_API int dmnerf_ins_label_rows_merged(const uint32_t* bitmaps, int world, const int32_t* labels, int64_t n, int ins_num,
                                            int32_t* gt_row, int32_t* n_valid, void* stream);
DMNERF_API int dmnerf_hungarian_partials(const float* pred, const int32_t* gt_row, int64_t n, int ins_num, double* partials,
                                         void* stream);
DMNERF_API int dmnerf_hungarian_costs_merged(const double* partials, int world, int64_t n_global, int ins_num, float* cost_ce,
                                             float* cost_siou, float* tp, float* col_sum, float* row_count, void* stream);

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
 * m = N*S).  out [M,C].  impl: DMNERF_IMPL_SIMT = exact fp32; DMNERF_IMPL_UMMA / AUTO = the tensor-core kernel, which also
 * keeps the ReLU masks (1 bit per unit) the gradient chain of the backward reads -- pass bit 0 of `flags` to
 * dmnerf_mlp_backward in that case.  The exact-fp32 kernel does not write the masks; the backward derives them from the saved
 * activations. */
DMNERF_API int dmnerf_mlp_forward_train(dmnerf_ctx* ctx, int net, const float* x, const float* rays_o, const float* rays_d,
                             const float* z, int64_t m, int s, float* out, float* acts, int impl, void* stream);

/* Gradient of a scalar loss w.r.t. the 30 parameters of network `net` given d_out = dL/d(out) [M,C] and the activations
 * saved by dmnerf_mlp_forward_train.  grads: 30 device buffers (state_dict order, parameter shapes), overwritten.
 * Gradient routing follows the reference (networks/dm_nerf.py:95: the instance branch reads h.detach()).
 * scratch: dmnerf_mlp_backward_scratch_floats(m) floats.  flags is a flag word: bit 0 = the forward wrote the ReLU bit planes
 * (tensor-core forward), bit 1 = the caller has already zero-filled `grads` (one fill instead of 30 memsets).
 * The heads are folded like in the forward, one masked split-bf16 wgmma GEMM per layer carries the gradient through the trunk
 * and batched wgmma GEMMs form the weight gradients, for any M. */
DMNERF_API int dmnerf_mlp_backward(dmnerf_ctx* ctx, int net, float* acts, const float* d_out, int64_t m, float* const* grads,
                        float* scratch, int flags, void* stream);

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
 * rows) is filled.  Of its input fields only `edit` is read; the others are ignored.
 * Deterministic path only (perturb = 0).  Synchronises the stream. */
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
 * last target after the occlusion fixes.  pieces (HOST, see "moving pieces" below): NULL is the reference's exchanger.
 *
 * ---- moving pieces (DESIGN.md, "Moving pieces"; no counterpart in the original) -------------------------------------------
 * A move may carry a region (a dmnerf_region, as in "region selection" below), so that only its label's samples inside that
 * piece move.  A sample of label mv at p = o + d z (fp32, the network prologue's
 * expression) is in the piece when the region does not drop it (the render kernels' per-sample test); mv must be among the
 * labels the region applies to.  A ray's accumulated label is the moving piece when it equals mv and the ray's vote is 1.
 * dmnerf_piece_vote: the votes of one fine pass: raw [N,S,C], its depths z [N,S], composite weights [N,S] and rays [N,3] ->
 *   votes [n_moves, N] (DEVICE uint8) = in >= out, where in (out) is the sum of w_s over the samples labelled move_labels[i]
 *   (argmax_sigmoid over all C - 4 channels) that the region keeps (drops), added in ascending sample order in fp32.  A move
 *   without a region (bits NULL) votes 1.  move_labels and regions are HOST arrays of n_moves.
 * dmnerf_exchanger with pieces: per move i with a region, the rays and this pass's depths of target i, the votes of the
 *   original rays and of target i's rays (their first fine pass), and rest_drop (1: the samples of mv outside the piece are
 *   zeroed, 0: kept); the original's rays and depths once.  A move whose region bits are NULL takes its whole label.  Every
 *   region is checked (dim in [2, 1290], finite map, mv among its labels, non-NULL votes, rays and depths) before any launch. */
#define DMNERF_MAX_MOVES 8
typedef struct dmnerf_pieces {
  dmnerf_region region[DMNERF_MAX_MOVES];       /* bits NULL: the move takes its whole label */
  int32_t rest_drop[DMNERF_MAX_MOVES];
  const uint8_t* ori_vote[DMNERF_MAX_MOVES];    /* [N] DEVICE: row i of the original rays' dmnerf_piece_vote */
  const uint8_t* tar_vote[DMNERF_MAX_MOVES];    /* [N] DEVICE: target i's vote for move i */
  const float* ori_rays_o;                      /* [N,3] DEVICE */
  const float* ori_rays_d;                      /* [N,3] */
  const float* ori_z;                           /* [N,S] the depths of ori_raw's samples */
  const float* tar_rays_o[DMNERF_MAX_MOVES];    /* [N,3] */
  const float* tar_rays_d[DMNERF_MAX_MOVES];    /* [N,3] */
  const float* tar_z[DMNERF_MAX_MOVES];         /* [N,S] the depths of tar_raws[i]'s samples */
} dmnerf_pieces;
DMNERF_API int dmnerf_exchanger(float* ori_raw, const float* const* tar_raws, const float* ori_acc, const float* const* tar_accs,
                                const int* move_labels, int n_moves, int64_t n, int s, int c, int64_t* ori_label,
                                int64_t* tar_label, const dmnerf_pieces* pieces, void* stream);
DMNERF_API int dmnerf_piece_vote(const float* raw, const float* z, const float* weights, const float* rays_o, const float* rays_d,
                                 int64_t n, int s, int c, const int* move_labels, const dmnerf_region* regions, int n_moves,
                                 uint8_t* votes, void* stream);

/* "Emptiness" regulariser on the per-sample object logits: emptiness_penalizer / ins_penalizer, networks/penalizer.py:5-62
 * (train_dmsr.py:53-60).  raw [n,S,C], z_vals [n,S], depth [n] (the rendered depth map, treated as a constant),
 * rays_d [n,3] -> loss[1] (device).  `partials` is caller-provided device scratch of dmnerf_penalizer_partials_bytes(n, S, C)
 * bytes.  The forward writes the mask populations and masked sums, summed in an order fixed by the sizes, into its head (the
 * first dmnerf_penalizer_state_bytes() bytes), which carries them to the backward call.  Backward (g_loss is a DEVICE scalar):
 * accumulate == 0 writes d_raw = g_loss[0] * dL/draw for EVERY channel (zeros in channels 0..3: no zero-fill needed);
 * accumulate != 0 adds the gradient to channels 4.. and leaves channels 0..3 untouched.
 * Over a batch split into W shards, every shard runs the forward on its rows (and ignores its loss), and
 * dmnerf_penalizer_merge adds the W gathered heads (`states`, W * dmnerf_penalizer_state_bytes() bytes, rank order) in rank
 * order -> `state` (the backward's state for the whole batch; the backward on it gives the shard's gradient) and loss[1].  At
 * W = 1 the merge gives the forward's own head and loss bit for bit. */
DMNERF_API int64_t dmnerf_penalizer_state_bytes(void);
DMNERF_API int64_t dmnerf_penalizer_partials_bytes(int64_t n, int s, int c);
DMNERF_API int dmnerf_penalizer_forward(const float* raw, const float* z_vals, const float* depth, const float* rays_d, int64_t n,
                                        int s, int c, float tolerance, float deta_w, void* partials, float* loss, void* stream);
DMNERF_API int dmnerf_penalizer_backward(const float* raw, const float* z_vals, const float* depth, const float* rays_d, int64_t n,
                                         int s, int c, float tolerance, float deta_w, const void* state, const float* g_loss,
                                         float* d_raw, int accumulate, void* stream);
DMNERF_API int dmnerf_penalizer_merge(const void* states, int world, int c, void* state, float* loss, void* stream);

/* dm_nerf(), networks/render.py:31-96, whole per-ray pipeline on device buffers. */
DMNERF_API int dmnerf_render_forward(dmnerf_ctx* ctx, const dmnerf_render_io* io, int64_t n_rays, int n_coarse,
                          int n_importance, int flags, int impl, void* stream);

/* ---- object selection (DESIGN.md, "Object selection") ----------------------------------------------------------------------
 * A bitmask of the KEPT object labels 0 .. ins_num, 4 uint32 words (bit k of word k / 32).  Every network sample gets the label
 * argmax(sigmoid(instance logits)) over all ins_num + 1 channels, first maximum winning (the exchanger's rule); a sample whose
 * label is not kept enters the composite with alpha = 0.  This applies to the coarse and the fine pass, so the coarse weights of
 * the selected scene drive the importance sampling.  raw_* (when asked for) stay the network's output.
 * dmnerf_render_forward(_host) and dmnerf_render_frame_host: io->edit->keep (fused kernel or stage kernels, chosen as without
 *   an edit).  A region or an appearance without keep keeps every label.
 * dmnerf_composite: keep_host (HOST, labels 0 .. c - 5; raw is read, not edited), NULL = no selection.
 * dmnerf_mesh_occupancy: keep_host (HOST), NULL = no selection; with one the rule applies per grid point (occ = 0 where the
 *   point's label is not kept) and labels (DEVICE int16 [dim^3], may be NULL) receives every point's label.  labels without
 *   keep_host is rejected.
 * Every one rejects a mask bit at or above ins_num + 1, naming the label. */

/* Same call with HOST buffers (pageable or pinned): copies rays in, renders, copies every non-NULL
 * output back, and synchronises the stream.  This is the end-to-end entry point bench.py times.
 * A batch of >= 131 072 rays is rendered in four parts (same bits: rays are independent) whose uploads / downloads travel on a
 * second stream while the neighbouring parts are rendered: only the first upload and the last download are exposed. */
DMNERF_API int dmnerf_render_forward_host(dmnerf_ctx* ctx, const dmnerf_render_io* io_host, int64_t n_rays, int n_coarse,
                               int n_importance, int flags, int impl, void* stream);

/* Synchronise `stream` and report any asynchronous failure of the kernels launched through `ctx` (CUDA errors and
 * the bounded-wait protocol checks of the tensor-core network kernels and backward GEMMs).  A protocol failure stays with the
 * weight set it ran with: later tensor-core launches through it refuse to start until the context is destroyed. */
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
 *   at a time (slab <= 0: 2^20), each slab reduced to occ = 1 - exp(-relu(sigma) * voxel) -> occ [dim,dim,dim].  keep_host /
 *   labels: the object selection and the label grid (see "object selection" above), both NULL for the whole scene.
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
                                     float voxel, int64_t slab, const uint32_t* keep_host, float* occ, int16_t* labels,
                                     void* stream);
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

/* ---- meshing an edited scene (DESIGN.md, "Meshing an edited scene"; no counterpart in the original) -------------------------
 * dmnerf_mesh_occupancy_edit: object moves applied per grid point to a labelled sweep.  occ / labels [dim^3] (DEVICE, in-out) hold
 *   the unedited keep-all sweep of network `net` on the grid of (transform_host, extents_host, dim) with this voxel; moves_host
 *   (HOST, n_moves in [0, DMNERF_MAX_MOVES]) are applied in order, each to the result of the previous ones.  Per move and grid
 *   point p (the sweep's fp32 point): t = trans p in fp64, rounded once to fp32; the network runs at t (zero view directions)
 *   only when its nearest grid index rint(A^-1 (t - b)) (the grid's index map, fp64) lies in the move's box.
 *   take = in box && label(t) == label && (occ(t) > level || occ_p <= level) && (no piece || the piece keeps t):
 *   (occ_p, label_p) = (occ(t), label).  Otherwise a point with label_p == label and occ_p > level that is in the piece (every
 *   point without a piece) or whose move has rest_drop gets occ_p = 0, its label kept.  slab <= 0: 2^20 points per slab.  evaluated_host (may be NULL) receives the number of
 *   target points evaluated.  Rejected on the host, before any launch: more than DMNERF_MAX_MOVES moves, a label outside
 *   [0, ins_num], a non-finite trans or one whose 3x3 part has det <= 0, a box outside the grid or inverted (the empty box
 *   (1, 0, 1, 0, 1, 0) is accepted and evaluates nothing), level outside (0, 1), a piece whose `applies` lacks the label.
 *   Synchronises the stream once per slab and move (the number of boxed points sizes the network launch).
 * dmnerf_mesh_vertex_labels: out [n] (DEVICE int16) = the label (labels, DEVICE int16 [dim^3]) of the solid grid point
 *   (occ > level) nearest to the index-space vertex verts [n,3] (DEVICE), among those closer than 2 (fp64 squared distances,
 *   ((dx^2 + dy^2) + dz^2)); an exact tie goes to the lowest linear index; -1 when there is none.  For a marching-cubes vertex of
 *   the same grid and level this is the inside end of its edge. */
typedef struct dmnerf_edit_move {
  int32_t label;
  int32_t rest_drop;          /* 1: the solid points of the label outside the piece are vacated too */
  double trans[12];           /* row-major 3x4 of the move, network frame: the edited scene shows at p what the network has at trans p */
  int32_t box[6];             /* inclusive index box (i_lo, i_hi, j_lo, j_hi, k_lo, k_hi) of the target points evaluated */
  dmnerf_region piece;        /* bits NULL: the whole label moves */
} dmnerf_edit_move;
DMNERF_API int dmnerf_mesh_occupancy_edit(dmnerf_ctx* ctx, int net, const double* transform_host, const double* extents_host, int dim,
                                          float voxel, float level, int64_t slab, const dmnerf_edit_move* moves_host, int n_moves,
                                          float* occ, int16_t* labels, int64_t* evaluated_host, void* stream);
DMNERF_API int dmnerf_mesh_vertex_labels(const float* verts, int64_t n, const float* occ, const int16_t* labels, int dim, float level,
                                         int16_t* out, void* stream);

/* ---- rendering moved objects per sample (DESIGN.md, "Rendering moved objects"; no counterpart in the original) ---------------
 * dmnerf_render_moved: dmnerf_render_forward's stage path (never the fused kernel) with the moves of dmnerf_mesh_occupancy_edit
 *   applied to the raw rows of each pass right after its network launch, before its composite.  Per move, in order, and sample
 *   p = o + d z (the network prologue's fp32 point) with raw row r_p and occupancy o_p = 1 - expf(-relu(r_p[3]) voxel): t and its
 *   nearest grid index as dmnerf_mesh_occupancy_edit computes them; the target's view direction trans[:3, :3] d (fp64, rounded
 *   once to fp32) normalised in fp32 as the prologue normalises d.  take = t's index in the box && label(t) == label &&
 *   (occ(t) > level || o_p <= level) && (no piece || the piece keeps t): r_p = the network's row at (t, its direction) (coarse
 *   network in the coarse pass, fine in the fine pass).  Otherwise, when label_p == label: r_p[3] = 0 (logits kept) if the piece
 *   keeps p (every p without one) and p's nearest index is in the box, or if rest_drop and the piece does not keep p.  The edited
 *   coarse weights drive the importance sampling; io->edit (selection, region, appearance) applies to the edited samples as in
 *   dmnerf_render_forward, and raw_* (when asked for) are the edited rows.  evaluated_host [2] (may be NULL): the targets
 *   evaluated in the coarse and the fine pass.  impl: DMNERF_IMPL_AUTO / _UMMA / _UMMA_F16 (the targets run on the same network).
 *   Rejected on the host, before any launch: everything dmnerf_mesh_occupancy_edit rejects of the grid, level and moves (n_moves in
 *   [1, DMNERF_MAX_MOVES], labels in [0, ins_num]), voxel not finite or <= 0, DMNERF_IMPL_SIMT and n (S + I) >= 2^31.  Reads the
 *   number of boxed targets back once per move and pass (synchronises the stream). */
typedef struct dmnerf_render_moves {
  const dmnerf_edit_move* moves;   /* HOST [n_moves] */
  int32_t n_moves;
  int32_t dim;                     /* the sweep grid the boxes index */
  double transform[16];            /* the sweep grid's scene transform, row-major */
  double extents[3];
  float level;                     /* (0, 1) */
  float voxel;                     /* > 0: the sweep's (far - near) / N_importance */
} dmnerf_render_moves;
DMNERF_API int dmnerf_render_moved(dmnerf_ctx* ctx, const dmnerf_render_io* io, int64_t n, int S, int NI, int flags, int impl,
                                   const dmnerf_render_moves* moves, int64_t* evaluated_host, void* stream);

/* ---- object inventory (DESIGN.md, "Object inventory"; no counterpart in the original) ---------------------------------------
 * Per-group reductions over the solid points (occ > level) of a grid occ [dim,dim,dim] (DEVICE, C order of the index (i, j, k)).
 * labels [dim^3] (DEVICE int16, may be NULL: every point is group 0) assigns each point its group 0 .. n_labels - 1.
 * boxes_host: HOST int32 [n_labels][6] = inclusive index boxes (i_lo, i_hi, j_lo, j_hi, k_lo, k_hi); with it only the solid
 * points inside their group's box count.  Every sum is an integer, so both calls are deterministic and independent of the launch
 * shape.  Both fail, before anything is written, when dim is outside [2, 2048], n_labels outside [1, 128], the grid holds NaN or
 * a label is outside [0, n_labels - 1].  One device->host read per call (synchronises the stream).
 * dmnerf_object_voxels: moments_host [n_labels][10] int64 = count, Si, Sj, Sk, Sii, Sjj, Skk, Sij, Sik, Sjk of the group's index
 *   coordinates; hist_host (may be NULL) [n_labels][3][dim] uint32 = its per-axis index histograms.  boxes_host may be NULL.
 * dmnerf_object_spans: axes_host [n_labels][3][4] fp64 (u0, u1, u2, o) -> spans_host [n_labels][3][2] = min and max over the
 *   group's points of s = ((u0 i + u1 j) + u2 k) + o, each operation rounded once in fp64; a group without points gets
 *   (+inf, -inf).  boxes_host is required. */
DMNERF_API int dmnerf_object_voxels(dmnerf_ctx* ctx, const float* occ, const int16_t* labels, int dim, float level, int n_labels,
                                    const int32_t* boxes_host, int64_t* moments_host, uint32_t* hist_host, void* stream);
DMNERF_API int dmnerf_object_spans(dmnerf_ctx* ctx, const float* occ, const int16_t* labels, int dim, float level, int n_labels,
                                   const int32_t* boxes_host, const double* axes_host, double* spans_host, void* stream);

/* ---- collision checks (DESIGN.md, "Collision checks"; no counterpart in the original) ----------------------------------------
 * Grid-only checks of object moves on a labelled keep-all sweep occ / labels [dim^3] (DEVICE float32 / int16, C order of the
 * index (i, j, k)) of the grid (transform_host, extents_host, dim); the network is not evaluated.  A point is solid when
 * occ > level.  Every count is an integer, so both calls are bit-reproducible and independent of the launch shape.  Both fail,
 * before anything is written, when the grid holds NaN or a label outside their range; one device->host read per call
 * (synchronises the stream).
 * dmnerf_move_overlap: each of the n_candidates moves (HOST, in [1, DMNERF_MAX_CANDIDATES]; fields as dmnerf_mesh_occupancy_edit,
 *   box = the source box B) is checked on its own against the grid.  Per grid point p (the sweep's fp32 point) and candidate:
 *   t = trans p in fp64, rounded once to fp32, q = rint(A^-1 (t - b)) as dmnerf_mesh_occupancy_edit computes them;
 *   src(p) = q in B && labels[q] == label && occ[q] > level && (no piece || the piece keeps t): the moved object covers p;
 *   obstacle(p) = occ[p] > level && labels[p] in obstacles_host (4 words of 32 labels; NULL: every label), except a point the
 *   move vacates (labels[p] == label and p in the piece -- every point without a piece -- or rest_drop).
 *   landed_host [n] (HOST int64) = #{p : src(p)}; overlap_host [n][128] (HOST int64) = #{p : src(p) && obstacle(p) &&
 *   labels[p] == l} per l.  Only the points of each candidate's destination box are visited: B grown by half a voxel, mapped
 *   back through the move, plus one voxel; this never changes a count.  Rejected on the host: dim outside [2, 2048], level
 *   outside (0, 1), a scene transform with det <= 0 or extents not finite and > 0, a candidate count out of range, and every
 *   candidate dmnerf_mesh_occupancy_edit rejects (labels in [0, 127]).  Fails on the device for a label outside [0, 127].
 * dmnerf_object_contacts: faces_host [3][n_labels][n_labels] (HOST int64) = per index axis a, #{p : solid l1 at p, solid l2 at
 *   p + e_a, l1 != l2}, never across a grid face.  Rejected: dim outside [2, 2048], n_labels outside [1, 128], level outside
 *   (0, 1); fails on the device for a label outside [0, n_labels - 1]. */
#define DMNERF_MAX_CANDIDATES 4096
DMNERF_API int dmnerf_move_overlap(dmnerf_ctx* ctx, const float* occ, const int16_t* labels, int dim, float level,
                                   const double* transform_host, const double* extents_host,
                                   const dmnerf_edit_move* candidates_host, int n_candidates, const uint32_t* obstacles_host,
                                   int64_t* overlap_host /* [n][128] */, int64_t* landed_host /* [n] */, void* stream);
DMNERF_API int dmnerf_object_contacts(dmnerf_ctx* ctx, const float* occ, const int16_t* labels, int dim, float level, int n_labels,
                                      int64_t* faces_host /* [3][n_labels][n_labels] */, void* stream);

/* ---- object placement (DESIGN.md, "Object placement"; no counterpart in the original) ---------------------------------------
 * Where object `label` (or its piece) comes to rest when it is lowered at every horizontal offset, from the labelled keep-all
 * sweep occ / labels [dim^3] (DEVICE float32 / int16, C order) of the grid (transform_host, extents_host, dim), in index space
 * and in integers: every result is bit-reproducible.  Heights y run along index axis `axis`, away from down: y = dim - 1 - idx
 * when sign is +1 (down is +e_axis), y = idx when sign is -1.  The horizontal axes (h1, h2) are the other two, ascending.
 *   object S:    labels[p] == label, occ[p] > level, and the piece keeps p's fp32 sweep point (every p without a piece);
 *   obstacles O: occ[p] > level, labels[p] in obstacles, and p not vacated (labels[p] == label and p in the piece -- every point
 *                without one -- or rest_drop), as dmnerf_move_overlap.
 * At offset (u, v) the object is raised by lift and lowered a voxel at a time: drop = -1 (blocked) when S + (u, v, lift)
 * overlaps O, otherwise the largest h such that no S + (u, v, lift - h') with h' in 0..h overlaps O or reaches below height 0.
 * At rest, contacts = the runs of S (maximal vertical runs of one column) whose bottom sits directly on an obstacle point, and
 * support = the obstacle label under the most of them (ties: the lowest label), -1 when there is none or the offset is blocked.
 * The offsets are those that keep S's horizontal index box inside the grid: u in [-h1_lo, dim - 1 - h1_hi], and as much for v.
 * The object lands at trans^-1 x for trans = translate(-A delta), delta the index displacement (dmnerf_move_overlap's convention).
 * Each call re-reads the grid: the grid check, a column pass that writes the column table (the highest obstacle height at or
 * below every height of every column, int16, in the context: 2 bytes per grid point, 2 GiB at dim 1024) and the object's runs.
 * Rejected on the host, before any launch: dim outside [2, 1024], level outside (0, 1), a scene transform with det <= 0 or
 * extents not finite and > 0, a label outside [0, 127], an axis outside {0, 1, 2}, a sign other than +-1, a lift outside
 * [0, dim - 1], a piece whose `applies` lacks the label.  After the one status read-back, before the map is computed: NaN in
 * occ, a label outside [0, 127] in labels, a label without solid points (in its piece), a lift that takes the object's top out
 * of the grid.
 * dmnerf_placement_map: drop, contacts (DEVICE int32) and support (DEVICE int16), each with room for dim * dim entries, receive
 *   the [U][V] row-major map; entry [i][j] is offset (offset_lo[0] + i, offset_lo[1] + j).  info_host gets the offsets, the
 *   object's height range, its runs, its points |S| and its sums over S of (h1, h2, y), so that its centre is exact.
 * dmnerf_placement_contacts: the support of one offset (u, v) inside the map's range: cells_host [n][3] (HOST int32, room for
 *   max_cells) = (h1 + u, h2 + v, label below) of every run resting on an obstacle, in (column, bottom) order of the runs;
 *   n_cells_host = n; drop_host = the map's drop there (no cells when it is -1).  Synchronises the stream. */
typedef struct dmnerf_placement {
  dmnerf_region piece;        /* bits NULL: the whole label is placed */
  uint32_t obstacles[4];      /* the labels that are obstacles, bit k of word k / 32 */
  int32_t label;
  int32_t rest_drop;          /* 1: the solid points of the label outside the piece are vacated too */
  int32_t axis;               /* the down axis: index axis 0, 1 or 2 */
  int32_t sign;               /* +1: down is +e_axis; -1: down is -e_axis */
  int32_t lift;               /* voxels the object is raised by before it is lowered */
} dmnerf_placement;
typedef struct dmnerf_placement_info {
  int32_t offset_lo[2];       /* the offset (u, v) of map entry [0][0] */
  int32_t offsets[2];         /* U, V */
  int32_t height[2];          /* the lowest and highest height of the object's points */
  int64_t runs;               /* its vertical runs */
  int64_t points;             /* |S| */
  int64_t sum[3];             /* sums over S of h1, h2 and y */
} dmnerf_placement_info;
DMNERF_API int dmnerf_placement_map(dmnerf_ctx* ctx, const float* occ, const int16_t* labels, int dim, float level,
                                    const double* transform_host, const double* extents_host, const dmnerf_placement* placement,
                                    int32_t* drop, int32_t* contacts, int16_t* support, dmnerf_placement_info* info_host, void* stream);
DMNERF_API int dmnerf_placement_contacts(dmnerf_ctx* ctx, const float* occ, const int16_t* labels, int dim, float level,
                                         const double* transform_host, const double* extents_host, const dmnerf_placement* placement,
                                         int u, int v, int32_t* cells_host, int64_t max_cells, int64_t* n_cells_host,
                                         int32_t* drop_host, void* stream);

/* ---- turned placements (DESIGN.md, "Turned placements"; no counterpart in the original) ------------------------------------
 * The placement of the object as a move `base` leaves it: base is a row-major 3x4 (fp64, network frame, as dmnerf_edit_move's
 * trans) and box_host [6] (HOST int32) the source box B (as dmnerf_move_overlap's box).  The object is S_base = {p : src(p)} with
 * src as dmnerf_move_overlap computes it: q = rint(A^-1 (t - b)) of t = fp32(base p) in B, labels[q] == label, occ[q] > level and
 * the piece keeps t; points carried outside the grid are lost.  The obstacles, heights, runs, drop, contacts, support and info are
 * dmnerf_placement_map's, taken over S_base; the obstacles are unchanged (the points the move vacates are the object's points as
 * it lies).  The placement at offset (u, v) with drop d is the move base translate(-A delta), delta as for dmnerf_placement_map:
 * the object lands at base^-1 x + A delta.  With base = I and the box of the label's solid points (grown by any margin), S_base
 * is dmnerf_placement_map's S and the maps are equal bit for bit.  Rejected on the host, before any launch: everything
 * dmnerf_placement_map rejects, a base that is not finite or has det <= 0, and a box outside the grid or inverted (the empty
 * box (1, 0, 1, 0, 1, 0) is accepted and leaves no point).
 * dmnerf_placement_maps: n_bases (in [1, DMNERF_MAX_BASES]) bases bases_host [n][12] in one call: the column table is built once,
 *   then per base the moved object's bytes (one reused buffer), its runs and its map.  drop, contacts, support (DEVICE, each with
 *   room for n * dim * dim entries): base i's [U_i][V_i] map starts at entry i * dim * dim.  status_host [n] (HOST int32) = 0
 *   placed, 1 no points after the move, 2 the object's top out of the grid at this lift; an unplaced base leaves its maps
 *   unwritten and its info_host [n] entry zero and does not fail the call.  The run buffers are sized from each base's point and
 *   run counts, so the call reads the status back once per base (synchronises the stream n times).
 * dmnerf_placement_contacts_moved: dmnerf_placement_contacts for the object as base_host [12] leaves it; fails when that base
 *   leaves no point or its top out of the grid. */
#define DMNERF_MAX_BASES 64
DMNERF_API int dmnerf_placement_maps(dmnerf_ctx* ctx, const float* occ, const int16_t* labels, int dim, float level,
                                     const double* transform_host, const double* extents_host, const dmnerf_placement* placement,
                                     const double* bases_host /* [n][12] */, const int32_t* box_host /* [6] */, int n_bases,
                                     int32_t* drop, int32_t* contacts, int16_t* support, dmnerf_placement_info* info_host /* [n] */,
                                     int32_t* status_host /* [n] */, void* stream);
DMNERF_API int dmnerf_placement_contacts_moved(dmnerf_ctx* ctx, const float* occ, const int16_t* labels, int dim, float level,
                                               const double* transform_host, const double* extents_host,
                                               const dmnerf_placement* placement, const double* base_host /* [12] */,
                                               const int32_t* box_host /* [6] */, int u, int v, int32_t* cells_host, int64_t max_cells,
                                               int64_t* n_cells_host, int32_t* drop_host, void* stream);

/* ---- arranging objects (DESIGN.md, "Arranging objects"; no counterpart in the original) -------------------------------------
 * dmnerf_grid_edit: the moves of dmnerf_mesh_occupancy_edit applied in order, in place, to the state occ / labels [dim^3] (DEVICE
 *   float32 / int16, in-out), with the network replaced by the source grid src_occ / src_labels [dim^3] (DEVICE, never written) at
 *   the target's nearest grid index: per move and state point p, t and q = rint(A^-1 (t - b)) as dmnerf_move_overlap computes
 *   them, take = q in B && src_labels[q] == label && (src_occ[q] > level || occ_p <= level) && (no piece || the piece keeps t):
 *   (occ_p, label_p) = (src_occ[q], label); otherwise dmnerf_mesh_occupancy_edit's vacate.  moves_host: n_moves in
 *   [1, DMNERF_MAX_MOVES], fields as dmnerf_mesh_occupancy_edit (labels in [0, 127]).  Per move: landed_host [n] (HOST int64) =
 *   the takes whose target is solid; overwritten_host [n][128] (HOST int64) = those of them that land on a solid state point of
 *   label l that the move does not vacate (label_p == label and p in the piece -- every point without one -- or rest_drop).  With
 *   the state equal to the source these are dmnerf_move_overlap's landed and overlap (every label an obstacle), and on a grid
 *   whose points and steps are exact in fp32 the result of whole-voxel translations and quarter turns is the edited sweep's.
 *   Every count is an integer and every write is per point, so the result is bit-reproducible.  Rejected on the host, before any
 *   launch: n_moves out of range, everything dmnerf_move_overlap rejects of the grid and the moves, and source and state buffers
 *   that overlap in memory.  Fails after the first read-back, with the state unwritten, on NaN or a label outside [0, 127] in
 *   either grid.  Two device->host reads: the grid checks, then the counts (synchronises the stream twice).
 * dmnerf_placement_maps_in_scene: dmnerf_placement_maps with the object S_base sampled from occ / labels and everything else --
 *   the obstacles, the points the move vacates, the labels under the resting runs -- taken from the scene scene_occ /
 *   scene_labels [dim^3] (DEVICE, the same grid).  The scene being occ / labels is dmnerf_placement_maps, bit for bit.  Both
 *   grids are checked.
 * dmnerf_placement_contacts_in_scene: dmnerf_placement_contacts_moved in the scene of dmnerf_placement_maps_in_scene. */
DMNERF_API int dmnerf_grid_edit(dmnerf_ctx* ctx, const float* src_occ, const int16_t* src_labels, int dim, float level,
                                const double* transform_host, const double* extents_host, const dmnerf_edit_move* moves_host, int n_moves,
                                float* occ, int16_t* labels, int64_t* landed_host /* [n] */, int64_t* overwritten_host /* [n][128] */,
                                void* stream);
DMNERF_API int dmnerf_placement_maps_in_scene(dmnerf_ctx* ctx, const float* occ, const int16_t* labels, const float* scene_occ,
                                              const int16_t* scene_labels, int dim, float level, const double* transform_host,
                                              const double* extents_host, const dmnerf_placement* placement,
                                              const double* bases_host /* [n][12] */, const int32_t* box_host /* [6] */, int n_bases,
                                              int32_t* drop, int32_t* contacts, int16_t* support,
                                              dmnerf_placement_info* info_host /* [n] */, int32_t* status_host /* [n] */, void* stream);
DMNERF_API int dmnerf_placement_contacts_in_scene(dmnerf_ctx* ctx, const float* occ, const int16_t* labels, const float* scene_occ,
                                                  const int16_t* scene_labels, int dim, float level, const double* transform_host,
                                                  const double* extents_host, const dmnerf_placement* placement,
                                                  const double* base_host /* [12] */, const int32_t* box_host /* [6] */, int u, int v,
                                                  int32_t* cells_host, int64_t max_cells, int64_t* n_cells_host, int32_t* drop_host,
                                                  void* stream);

/* ---- copying objects (DESIGN.md, "Copying objects"; no counterpart in the original) ----------------------------------------
 * A copy is a move that leaves its source in place: it takes exactly as the move with the same fields takes (same target, box,
 * piece test and air clause) and writes the source's label, and it never vacates.  The entry points below are the ones they are
 * named after with copy flags: copies_host [n] (HOST int32, one per move or candidate; NULL: none) or `copy` (one per call),
 * each 0 or 1.  With every flag 0 each equals its namesake bit for bit.
 * dmnerf_mesh_occupancy_edit_copies, dmnerf_grid_edit_copies, dmnerf_render_moved_copies: a copy skips the vacate.  In
 *   dmnerf_grid_edit_copies a copy's overwritten_host counts every solid state point it lands on, its own label's included.
 * dmnerf_move_overlap_copies: a copy candidate's own label's solid points are obstacles like any other (with or without a
 *   piece).  The candidates are grouped by kind on the host, one launch per kind; the results stay in the caller's order.
 * dmnerf_placement_maps_in_scene_copy, dmnerf_placement_contacts_in_scene_copy: with copy, the scene's solid points of the label
 *   are obstacles (the object's source stays where it is).
 * Rejected on the host, before any launch, beside everything the namesake rejects: a flag other than 0 or 1, a copy with
 * rest_drop (a copy vacates nothing), and, for the moves applied in order (not dmnerf_move_overlap_copies' independent
 * candidates), a move of a label after a copy of it (its vacate would erase the copy, which carries the label). */
DMNERF_API int dmnerf_mesh_occupancy_edit_copies(dmnerf_ctx* ctx, int net, const double* transform_host, const double* extents_host,
                                                 int dim, float voxel, float level, int64_t slab, const dmnerf_edit_move* moves_host,
                                                 const int32_t* copies_host /* [n] */, int n_moves, float* occ, int16_t* labels,
                                                 int64_t* evaluated_host, void* stream);
DMNERF_API int dmnerf_grid_edit_copies(dmnerf_ctx* ctx, const float* src_occ, const int16_t* src_labels, int dim, float level,
                                       const double* transform_host, const double* extents_host, const dmnerf_edit_move* moves_host,
                                       const int32_t* copies_host /* [n] */, int n_moves, float* occ, int16_t* labels,
                                       int64_t* landed_host /* [n] */, int64_t* overwritten_host /* [n][128] */, void* stream);
DMNERF_API int dmnerf_render_moved_copies(dmnerf_ctx* ctx, const dmnerf_render_io* io, int64_t n, int S, int NI, int flags, int impl,
                                          const dmnerf_render_moves* moves, const int32_t* copies_host /* [n_moves] */,
                                          int64_t* evaluated_host, void* stream);
DMNERF_API int dmnerf_move_overlap_copies(dmnerf_ctx* ctx, const float* occ, const int16_t* labels, int dim, float level,
                                          const double* transform_host, const double* extents_host,
                                          const dmnerf_edit_move* candidates_host, const int32_t* copies_host /* [n] */,
                                          int n_candidates, const uint32_t* obstacles_host, int64_t* overlap_host /* [n][128] */,
                                          int64_t* landed_host /* [n] */, void* stream);
DMNERF_API int dmnerf_placement_maps_in_scene_copy(dmnerf_ctx* ctx, const float* occ, const int16_t* labels, const float* scene_occ,
                                                   const int16_t* scene_labels, int dim, float level, const double* transform_host,
                                                   const double* extents_host, const dmnerf_placement* placement, int copy,
                                                   const double* bases_host /* [n][12] */, const int32_t* box_host /* [6] */,
                                                   int n_bases, int32_t* drop, int32_t* contacts, int16_t* support,
                                                   dmnerf_placement_info* info_host /* [n] */, int32_t* status_host /* [n] */,
                                                   void* stream);
DMNERF_API int dmnerf_placement_contacts_in_scene_copy(dmnerf_ctx* ctx, const float* occ, const int16_t* labels, const float* scene_occ,
                                                       const int16_t* scene_labels, int dim, float level, const double* transform_host,
                                                       const double* extents_host, const dmnerf_placement* placement, int copy,
                                                       const double* base_host /* [12] */, const int32_t* box_host /* [6] */, int u,
                                                       int v, int32_t* cells_host, int64_t max_cells, int64_t* n_cells_host,
                                                       int32_t* drop_host, void* stream);

/* ---- moving objects together (DESIGN.md, "Moving objects together"; no counterpart in the original) -------------------------
 * A move may carry a label set G (a table and what stands on it) that holds its own label: each rule tests "label in G" where a
 * move of one label tests "label == label".  The take writes the target's own label; the vacate clears the points of every label
 * of G (with the piece and rest_drop tests of a single move); the piece (region_drops) is evaluated for the label of the point
 * tested, so a piece cuts the labels of G it applies to and the others move whole.  A label outside [0, 127] (a state grid of
 * dmnerf_mesh_occupancy_edit is not checked) belongs to no set, as it equalled no move's label before.  The collision checks do not count the points
 * a group vacates; placement places the solid points of G (the piece applied) as one body, and a copy keeps its source's points
 * as obstacles.  The entry points below are the _copies / _copy ones with label sets: groups_host [n][4] (HOST uint32, the label
 * words of each move or candidate, bit k of word k / 32; NULL: each move's own label) or group_host [4] (one per call; NULL: the
 * placement's label).  With every set {label} each equals its namesake bit for bit; a group is one move towards
 * DMNERF_MAX_MOVES and evaluates its targets in one pass.
 * Rejected on the host, before any launch, beside everything the namesake rejects: a set without its move's label, a set with a
 * label outside [0, ins_num] (outside [0, 127] for the grid-only calls: dmnerf_grid_edit_groups, dmnerf_move_overlap_groups and
 * the placement pair), and, for the moves applied in order, a move whose set holds a label of an earlier copy's set.  Each error
 * names the entry point called. */
DMNERF_API int dmnerf_mesh_occupancy_edit_groups(dmnerf_ctx* ctx, int net, const double* transform_host, const double* extents_host,
                                                 int dim, float voxel, float level, int64_t slab, const dmnerf_edit_move* moves_host,
                                                 const int32_t* copies_host /* [n] */, const uint32_t* groups_host /* [n][4] */,
                                                 int n_moves, float* occ, int16_t* labels, int64_t* evaluated_host, void* stream);
DMNERF_API int dmnerf_grid_edit_groups(dmnerf_ctx* ctx, const float* src_occ, const int16_t* src_labels, int dim, float level,
                                       const double* transform_host, const double* extents_host, const dmnerf_edit_move* moves_host,
                                       const int32_t* copies_host /* [n] */, const uint32_t* groups_host /* [n][4] */, int n_moves,
                                       float* occ, int16_t* labels, int64_t* landed_host /* [n] */,
                                       int64_t* overwritten_host /* [n][128] */, void* stream);
DMNERF_API int dmnerf_render_moved_groups(dmnerf_ctx* ctx, const dmnerf_render_io* io, int64_t n, int S, int NI, int flags, int impl,
                                          const dmnerf_render_moves* moves, const int32_t* copies_host /* [n_moves] */,
                                          const uint32_t* groups_host /* [n_moves][4] */, int64_t* evaluated_host, void* stream);
DMNERF_API int dmnerf_move_overlap_groups(dmnerf_ctx* ctx, const float* occ, const int16_t* labels, int dim, float level,
                                          const double* transform_host, const double* extents_host,
                                          const dmnerf_edit_move* candidates_host, const int32_t* copies_host /* [n] */,
                                          const uint32_t* groups_host /* [n][4] */, int n_candidates, const uint32_t* obstacles_host,
                                          int64_t* overlap_host /* [n][128] */, int64_t* landed_host /* [n] */, void* stream);
DMNERF_API int dmnerf_placement_maps_in_scene_group(dmnerf_ctx* ctx, const float* occ, const int16_t* labels, const float* scene_occ,
                                                    const int16_t* scene_labels, int dim, float level, const double* transform_host,
                                                    const double* extents_host, const dmnerf_placement* placement, int copy,
                                                    const uint32_t* group_host /* [4] */, const double* bases_host /* [n][12] */,
                                                    const int32_t* box_host /* [6] */, int n_bases, int32_t* drop, int32_t* contacts,
                                                    int16_t* support, dmnerf_placement_info* info_host /* [n] */,
                                                    int32_t* status_host /* [n] */, void* stream);
DMNERF_API int dmnerf_placement_contacts_in_scene_group(dmnerf_ctx* ctx, const float* occ, const int16_t* labels,
                                                        const float* scene_occ, const int16_t* scene_labels, int dim, float level,
                                                        const double* transform_host, const double* extents_host,
                                                        const dmnerf_placement* placement, int copy,
                                                        const uint32_t* group_host /* [4] */, const double* base_host /* [12] */,
                                                        const int32_t* box_host /* [6] */, int u, int v, int32_t* cells_host,
                                                        int64_t max_cells, int64_t* n_cells_host, int32_t* drop_host, void* stream);

/* ---- Deforming objects (DESIGN.md, "Deforming objects") ----------------------------------------------------------------------
 * A move may bend, twist and taper its object: a height-preserving deformation D of the object where it stands, before the move,
 * so that the forward map is x -> trans^-1 D(x) and a destination point p shows the network at x = D^-1(trans p).  D acts in a
 * frame of the network frame: centre c and orthonormal right-handed axes e_u, e_v, e_h (e_h "up"); in frame coordinates
 * (u, v, h) it maps (u, v) -> A(h) (u, v) + t(h) and keeps h, A(h) and t(h) interpolating n_knots knots linearly at heights
 * h0 + k dh, clamped to the end knots outside them.  frame: the rows e_u, e_v, e_h, c; knots: HOST double [n_knots][6], A row-major
 * then t.  n_knots == 0: a rigid move (every other field ignored).  The pull is fp64 with one rounding per operation and rounded once
 * to fp32 before the existing box test; the moved render's view direction is the pulled-back ray's tangent.
 * The entry points below are the _groups ones with deformations_host [n] (HOST; NULL: every move rigid).  An all-rigid array
 * equals the namesake bit for bit.  Rejected on the host before any launch, with an error naming the entry point: n_knots outside
 * {0} and [2, 64], NULL knots, a non-finite value, dh <= 0, a frame that is not orthonormal and right-handed to 1e-9, and
 * det A(h) <= 0 anywhere on a knot interval. */
typedef struct dmnerf_deformation {
  int32_t n_knots;            /* 0: rigid; otherwise in [2, 64] */
  double frame[12];           /* e_u, e_v, e_h, c (network frame) */
  double h0, dh;              /* knot k at height h0 + k dh, dh > 0 */
  const double* knots;        /* HOST [n_knots][6]: A00 A01 A10 A11 t0 t1 */
} dmnerf_deformation;
DMNERF_API int dmnerf_mesh_occupancy_edit_deformed(dmnerf_ctx* ctx, int net, const double* transform_host, const double* extents_host,
                                                   int dim, float voxel, float level, int64_t slab, const dmnerf_edit_move* moves_host,
                                                   const int32_t* copies_host /* [n] */, const uint32_t* groups_host /* [n][4] */,
                                                   const dmnerf_deformation* deformations_host /* [n] */, int n_moves, float* occ,
                                                   int16_t* labels, int64_t* evaluated_host, void* stream);
DMNERF_API int dmnerf_grid_edit_deformed(dmnerf_ctx* ctx, const float* src_occ, const int16_t* src_labels, int dim, float level,
                                         const double* transform_host, const double* extents_host, const dmnerf_edit_move* moves_host,
                                         const int32_t* copies_host /* [n] */, const uint32_t* groups_host /* [n][4] */,
                                         const dmnerf_deformation* deformations_host /* [n] */, int n_moves, float* occ,
                                         int16_t* labels, int64_t* landed_host /* [n] */, int64_t* overwritten_host /* [n][128] */,
                                         void* stream);
DMNERF_API int dmnerf_render_moved_deformed(dmnerf_ctx* ctx, const dmnerf_render_io* io, int64_t n, int S, int NI, int flags, int impl,
                                            const dmnerf_render_moves* moves, const int32_t* copies_host /* [n_moves] */,
                                            const uint32_t* groups_host /* [n_moves][4] */,
                                            const dmnerf_deformation* deformations_host /* [n_moves] */, int64_t* evaluated_host,
                                            void* stream);
DMNERF_API int dmnerf_move_overlap_deformed(dmnerf_ctx* ctx, const float* occ, const int16_t* labels, int dim, float level,
                                            const double* transform_host, const double* extents_host,
                                            const dmnerf_edit_move* candidates_host, const int32_t* copies_host /* [n] */,
                                            const uint32_t* groups_host /* [n][4] */,
                                            const dmnerf_deformation* deformations_host /* [n] */, int n_candidates,
                                            const uint32_t* obstacles_host, int64_t* overlap_host /* [n][128] */,
                                            int64_t* landed_host /* [n] */, void* stream);

/* ---- connected components (DESIGN.md, "Connected components"; no counterpart in the original) --------------------------------
 * The solid points (occ > level) of a grid occ [dim,dim,dim] (DEVICE, C order, p = (i dim + j) dim + k) split into components:
 * two solid points are adjacent when they are face neighbours (connectivity 6) or face, edge or corner neighbours (26), never
 * across a grid face, and, with labels (DEVICE int16, may be NULL), carry the same label.  A component's root is its smallest p;
 * components are numbered 0 .. n - 1 in ascending root order, so every result is canonical and bit-reproducible.  dim must be in
 * [2, 1290] (dim^3 < 2^31).  Each call validates on the device and reads back once (synchronises the stream) before anything is
 * reported.
 * dmnerf_object_components: comp [dim^3] (DEVICE int32) = the point's component id, or -1 where not solid; n_components_host =
 *   n.  Fails when n_labels is outside [1, 128], connectivity is not 6 or 26, the grid holds NaN or a label (of any point) is
 *   outside [0, n_labels - 1].
 * dmnerf_component_table: per component of comp (n components) label [n] (DEVICE int16; 0 without labels), voxels [n] and
 *   root [n] (DEVICE int64).  Fails when comp holds an id outside [-1, n).
 * dmnerf_component_groups: groups [dim^3] (DEVICE int16) = lut[comp[p]] (lut: DEVICE int16 [n]), or `discard` where comp is -1;
 *   the group grid of the inventory entry points above.  Fails when comp holds an id outside [-1, n). */
DMNERF_API int dmnerf_object_components(dmnerf_ctx* ctx, const float* occ, const int16_t* labels, int dim, float level, int n_labels,
                                        int connectivity, int32_t* comp, int64_t* n_components_host, void* stream);
DMNERF_API int dmnerf_component_table(dmnerf_ctx* ctx, const int32_t* comp, const int16_t* labels, int dim, int64_t n, int16_t* label,
                                      int64_t* voxels, int64_t* root, void* stream);
DMNERF_API int dmnerf_component_groups(dmnerf_ctx* ctx, const int32_t* comp, int dim, int64_t n, const int16_t* lut, int discard,
                                       int16_t* groups, void* stream);

/* ---- viewing the labelled grid (DESIGN.md, "Viewing the labelled grid"; no counterpart in the original) ----------------------
 * dmnerf_grid_cast: per ray the first solid, kept voxel of a labelled grid occ [dim^3] (DEVICE float32) / labels [dim^3] (DEVICE
 *   int16), with the scene transform and extents of the sweep (HOST float64, as dmnerf_mesh_occupancy), dim in [2, 1290].  Grid
 *   point q owns the cube [q - 1/2, q + 1/2]^3; the ray o + t d (rays_o, rays_d [n][3], DEVICE float32, network frame; t in the
 *   units of d as given) is cast over t in [near, far] clipped to the grid's cube [-1/2, dim - 1/2]^3 in index space
 *   (u(t) = inv (o - b) + t inv d with the index map of dmnerf_mesh_occupancy_edit) by a voxel walk whose boundary times are
 *   computed directly in fp64, one rounding per operation, ties stepping i before j before k.  A voxel is solid when
 *   occ > level (NaN never is) and, with keep_words_host (HOST uint32 [4], may be NULL: every label), its label is in [0, 127]
 *   and kept.  Per ray: t_out (DEVICE float32) = the hit voxel's entry time max(t0, t_entry) rounded once, +inf without a hit;
 *   label_out (DEVICE int16) and voxel_out (DEVICE int32, C-order linear index) = -1 without a hit; normal_out [n][3] (DEVICE
 *   float32, may be NULL) = -inv^T grad(occ) at the voxel normalised (central differences, one-sided at the grid's faces),
 *   the entry face's normal when that gradient is zero or not finite, -d / |d| when the ray starts inside the voxel; 0 without
 *   a hit.  Rays with a non-finite or zero direction, or that miss the grid, have no hit.  No atomics and no read-back: the
 *   call does not synchronise and repeats bit for bit.  Rejected on the host before any launch, writing nothing: NULL grid, transform
 *   or extents, NULL ray or output pointers with n > 0, dim out of range, a non-finite level, near / far not finite or
 *   near > far, n < 0, a transform that is not finite or has det <= 0, extents not finite and > 0. */
DMNERF_API int dmnerf_grid_cast(dmnerf_ctx* ctx, const float* occ, const int16_t* labels, int dim, float level,
                                const double* transform_host, const double* extents_host, const uint32_t* keep_words_host,
                                const float* rays_o, const float* rays_d, int64_t n, float near_t, float far_t, float* t_out,
                                int16_t* label_out, int32_t* voxel_out, float* normal_out, void* stream);
/* dmnerf_grid_edit_source: where each hit of dmnerf_grid_cast on an edited grid came from (DESIGN.md, "Viewing the labelled grid",
 *   "Colouring an edited view").  occ / labels [dim^3] (DEVICE) is the viewed grid, src_occ / src_labels [dim^3] (DEVICE, separate
 *   memory) the unedited source, and moves (with copies_host [n_moves], groups_host [n_moves][4] and deformations_host [n_moves],
 *   each HOST and may be NULL, as dmnerf_render_moved_deformed) the edit; moves->dim, transform, extents and level give the grid.
 *   rays_o / rays_d [n][3] and t_out / voxel_out [n] (DEVICE) are the cast's rays and outputs.  Per ray with voxel q >= 0 the
 *   moves of dmnerf_grid_edit are replayed at q's sweep point alone, from (src_occ[q], src_labels[q]), with that call's take and
 *   vacate; move_out [n] (DEVICE int32) = the last move that took (-1: none, or no hit).  The replay's result must equal
 *   (occ[q], labels[q]), the occupancy by its bits: *mismatched_host (HOST int64) = the hits where it does not.  x = o + t d (fp32,
 *   multiply then add).  point_out [n][3] (DEVICE float32) = the target of x under move_out (edit_target, pulled through its
 *   deformation), x where no move took, NaN without a hit; dir_out [n][3] (DEVICE float32) = trans[:3, :3] d in fp64 (pulled back
 *   by the deformation's tangent at x's pulled point), rounded once, not normalised; d where no move took; 0 without a hit.
 *   Rejected on the host before any launch: everything dmnerf_render_moved_deformed rejects of the moves (labels in [0, 127]),
 *   dim above 1290, NULL pointers, n < 0, source and viewed grids that overlap.  One read-back (synchronises the stream); fails
 *   after it when a voxel index lies outside [-1, dim^3). */
DMNERF_API int dmnerf_grid_edit_source(dmnerf_ctx* ctx, const float* occ, const int16_t* labels, const float* src_occ,
                                       const int16_t* src_labels, const dmnerf_render_moves* moves, const int32_t* copies_host,
                                       const uint32_t* groups_host, const dmnerf_deformation* deformations_host, const float* rays_o,
                                       const float* rays_d, const float* t_out, const int32_t* voxel_out, int64_t n,
                                       int32_t* move_out, float* point_out, float* dir_out, int64_t* mismatched_host, void* stream);

/* ---- region selection (DESIGN.md, "Region selection"; no counterpart in the original) ------------------------------------
 * A region (dmnerf_region) is one bit per point of a sweep grid [dim,dim,dim] (dim in [2, 1290]; point v = (i dim + j) dim + k
 * is bit v & 31 of word v >> 5, ceil(dim^3 / 32) uint32 words, the bits past dim^3 zero), the voxel map [M | c] (row-major 3x4
 * float32, network frame -> grid index), the labels it applies to (4 words, as a keep mask) and the rule for samples outside the
 * grid.  A render sample at p = o + d z (fp32, as the network prologue computes it) with label l (argmax_sigmoid, as object
 * selection) gets alpha = 0 when l is in `applies` and either p's nearest grid point (i_a = rint(((M_a0 p0 + M_a1 p1) + M_a2 p2)
 * + c_a), every operation rounded once) is inside the grid with bit 0, or p is outside it and outside_keep is 0.  NaN and inf
 * are outside.
 * dmnerf_render_forward(_host) and dmnerf_render_frame_host: io->edit->region (fused kernels or stage kernels, chosen as without
 *   an edit; with or without keep).  The render fails for NULL bits, dim out of range, a non-finite map or `applies` holding a
 *   label above the bound networks' ins_num.
 * dmnerf_region_pack: bits (DEVICE) = for every point, the bit of its id in table (DEVICE uint32, bit id of word id / 32, over
 *   ids 0 .. n_ids - 1); an id outside [0, n_ids) (-1: no component) gives 0.  ids: DEVICE int32 [dim^3].
 * dmnerf_region_dilate: out = `radius` steps of binary dilation of in (6: face neighbours, 26: also edge and corner neighbours;
 *   never across a grid face; radius 0 copies), then the complement when invert != 0 (tail bits stay 0).  in and out are
 *   distinct DEVICE buffers.
 * dmnerf_region_contains: out [n] (DEVICE uint8) = 1 where the point pts [n,3] (DEVICE) is inside the grid of `region` (bits,
 *   dim and voxel map are read) and its bit is 1: the render kernels' own test. */
DMNERF_API int dmnerf_region_pack(const int32_t* ids, int dim, const uint32_t* table, int64_t n_ids, uint32_t* bits, void* stream);
DMNERF_API int dmnerf_region_dilate(dmnerf_ctx* ctx, const uint32_t* in, int dim, int radius, int connectivity, int invert,
                                    uint32_t* out, void* stream);
DMNERF_API int dmnerf_region_contains(const dmnerf_region* region, const float* pts, int64_t n, uint8_t* out, void* stream);

/* ---- object appearance (DESIGN.md, "Object appearance"; no counterpart in the original) -----------------------------------
 * An appearance is one row of 16 floats per label l in [0, ins_num]: the colour map [M_l | b_l] (row-major 3x4), the density
 * scale s_l (finite, >= 0) and 3 floats of padding (finite, ignored).  The identity row is [I | 0], s = 1.  A render sample with
 * label l (argmax_sigmoid, as object selection) that the selection and the region keep gets alpha = 1 - expf(-(s_l max(sigma,
 * 0)) dist) and the colour c'_a = min(max(((M_a0 c0 + M_a1 c1) + M_a2 c2) + b_a, 0), 1) of its sigmoid colour c, every
 * operation rounded once in fp32; a dropped sample keeps alpha = 0.  Depth, acc and the instance maps use the edited weights,
 * raw_* stay the network's output, and the coarse weights of the edited scene drive the importance sampling.
 * dmnerf_render_forward(_host) and dmnerf_render_frame_host: io->edit->appearance with appearance_labels rows (fused kernels or
 *   stage kernels, chosen as without an edit; with or without keep and a region).  The table is copied on the call's stream into
 *   the context once per call, so it may be freed on return.  The render fails for appearance_labels outside
 *   [2, DMNERF_MAX_INS + 1] or other than the bound networks' ins_num + 1, an entry that is not finite or a negative scale. */

/* ---- test-view evaluation: render_test, networks/tester.py (+ ins_eval / calculate_ap, networks/evaluator.py:77-175) -------
 * Rules and deviations: DESIGN.md, "Evaluation metrics".  Every result is deterministic (fixed-order reductions, integer atomics
 * only).  `res` is DEVICE memory; reading it back is the caller's one device->host transfer per frame.  `ws` is caller-provided
 * device scratch of dmnerf_eval_workspace_bytes(n, k, H, W) bytes, shared by both calls (stream-ordered).
 *
 * dmnerf_eval_image: PSNR (skimage 0.18.3 peak_signal_noise_ratio, data_range 1: fp32 difference and square, fp64 mean) and SSIM
 *   (structural_similarity, multichannel, data_range 1: 7x7 uniform filter in fp64, mean over the interior cropped by 3, mean of
 *   the channels) of rgb vs gt [H,W,3] float32 -> res->psnr, res->ssim.  H and W must be >= 7.
 * dmnerf_ins_eval: ins_eval of the instance map ins [n,k] float32 against gt ranks gt_row [n] int32 (rank in [0, gt_num), anything
 *   else = no gt object).  Mask (crop path): a pixel is masked where mask[i] == 0 (mask: float32 [n]) or mask_labels[i] >=
 *   mask_below (mask_labels: int32 [n]); at most one of the two is non-NULL.  Writes pred_label [n] int64 (first maximum, k where
 *   masked) and res->ap, gt_num, pred_num, return_labels[0..gt_num), status (0 ok, 1 NaN in the instance map).
 * dmnerf_calculate_ap: calculate_ap(ious, gt_number, confidence, 'integral') of m <= 128 matches (conf may be NULL: ordered by
 *   IoU) -> ap6 [6] float32 (device).
 * dmnerf_ins_dense_rows: one-hot gt_ins [n,k] float32 -> rank of the first non-zero column among the first gt_num, or -1.
 * dmnerf_label_colors: out [n,3] uint8 = lut[labels[i]] (lut [n_lut,3] uint8, device), black outside [0, n_lut); labels int64 when
 *   labels_are_64bit, otherwise int32. */
typedef struct dmnerf_eval_result {
  float ap[6];                      /* AP50, AP75, AP80, AP85, AP90, AP95 */
  int32_t gt_num, pred_num, status, reserved;
  double psnr, ssim;
  int32_t return_labels[DMNERF_MAX_INS + 1];   /* matched predicted label per gt object, or -1 */
} dmnerf_eval_result;
DMNERF_API int64_t dmnerf_eval_workspace_bytes(int64_t n, int k, int H, int W);
DMNERF_API int dmnerf_eval_image(const float* rgb, const float* gt, int H, int W, void* ws, dmnerf_eval_result* res, void* stream);
DMNERF_API int dmnerf_ins_eval(const float* ins, int64_t n, int k, const int32_t* gt_row, int gt_num, const float* mask,
                               const int32_t* mask_labels, int mask_below, int64_t* pred_label, void* ws, dmnerf_eval_result* res,
                               void* stream);
DMNERF_API int dmnerf_calculate_ap(const float* ious, const float* conf, int m, int gt_number, float* ap6, void* stream);
DMNERF_API int dmnerf_ins_dense_rows(const float* gt_ins, int64_t n, int k, int gt_num, int32_t* gt_row, void* stream);
DMNERF_API int dmnerf_label_colors(const void* labels, int labels_are_64bit, int64_t n, const uint8_t* lut, int n_lut, uint8_t* out,
                                   void* stream);

/* Number of kernels this library has launched on the calling thread's contexts since load. */
DMNERF_API int64_t dmnerf_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* DMNERF_B200_H_ */
