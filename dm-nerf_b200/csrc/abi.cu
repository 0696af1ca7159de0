// extern "C" boundary of libdmnerf_b200.so: context, weight binding, stage entry points and the
// whole-pipeline render call.  See include/dmnerf_b200.h for the contract of every symbol.
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "umma_api.cuh"

namespace dmnerf {

static thread_local std::string g_error;
std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_error = buf;
}

// Grow-only device scratch buffer.
struct Scratch {
  void* ptr = nullptr;
  size_t cap = 0;
  int reserve(size_t bytes) {
    if (bytes <= cap) return 0;
    if (ptr) DMN_CUDA(cudaFree(ptr));
    ptr = nullptr; cap = 0;
    const size_t want = bytes + bytes / 4;
    DMN_CUDA(cudaMalloc(&ptr, want));
    cap = want;
    return 0;
  }
  void release() { if (ptr) cudaFree(ptr); ptr = nullptr; cap = 0; }
};

}  // namespace dmnerf

using namespace dmnerf;

constexpr int HOST_PARTS = 4;              // a *_host call on >= HOST_PART_MIN_RAYS rays is rendered in this many parts
constexpr int64_t HOST_PART_MIN_RAYS = 131072;

struct dmnerf_ctx {
  int device = 0;
  NetParams net[2];
  UmmaWeights packed[2];          // tensor-core operand images (umma_api.cuh)
  Scratch ws_raw_c, ws_raw_f, ws_z_c, ws_z_f, ws_w_c, ws_w_f;
  Scratch host_in, host_out;      // device staging for the *_host entry point
  Scratch frame_rays;             // rays of the frame being rendered by dmnerf_render_frame_host
  Scratch mesh_pts, mesh_raw;     // one slab of the occupancy sweep: points + zero view directions, network output
  MeshState* mesh = nullptr;      // buffers of the other mesh entry points (mesh.cu)
  bool train_feats_missing[2] = {false, false};
  bool profiling = false;
  bool last_fused = false;       // the last render call took the single-kernel path
  bool profile_valid = false;
  cudaEvent_t ev[DMNERF_N_STAGES + 1] = {};
  // *_host entry points: second stream + events so that the copies of one part of a large batch overlap the kernels of the next
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_in[HOST_PARTS] = {}, ev_done[HOST_PARTS] = {}, ev_start = nullptr;
  dmnerf_ctx() { memset(net, 0, sizeof(net)); }
};

extern "C" {

DMNERF_API int dmnerf_abi_version(void) { return DMNERF_ABI_VERSION; }
DMNERF_API const char* dmnerf_last_error(void) { return g_error.c_str(); }
DMNERF_API int64_t dmnerf_launch_count(void) { return g_launches.load(); }

DMNERF_API int dmnerf_ctx_create(int device, dmnerf_ctx** out) {
  DMN_CHECK(out != nullptr, "ctx_create: out is NULL");
  *out = nullptr;
  int count = 0;
  DMN_CUDA(cudaGetDeviceCount(&count));
  DMN_CHECK(device >= 0 && device < count, "ctx_create: device %d not in [0,%d)", device, count);
  DMN_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  DMN_CUDA(cudaGetDeviceProperties(&prop, device));
  DMN_CHECK(prop.major == 9 && prop.minor == 0, "ctx_create: this library is built for sm_90a only (device is sm_%d%d)", prop.major, prop.minor);
  dmnerf_ctx* c = new dmnerf_ctx();
  c->device = device;
  *out = c;
  return 0;
}

DMNERF_API int dmnerf_ctx_destroy(dmnerf_ctx* ctx) {
  if (!ctx) return 0;
  cudaSetDevice(ctx->device);
  for (int i = 0; i < 2; ++i) umma_weights_free(ctx->packed[i]);
  Scratch* all[] = {&ctx->ws_raw_c, &ctx->ws_raw_f, &ctx->ws_z_c, &ctx->ws_z_f, &ctx->ws_w_c, &ctx->ws_w_f,
                    &ctx->host_in, &ctx->host_out, &ctx->frame_rays, &ctx->mesh_pts, &ctx->mesh_raw};
  for (Scratch* s : all) s->release();
  mesh_state_free(ctx->mesh);
  for (cudaEvent_t e : ctx->ev) if (e) cudaEventDestroy(e);
  for (cudaEvent_t e : ctx->ev_in) if (e) cudaEventDestroy(e);
  for (cudaEvent_t e : ctx->ev_done) if (e) cudaEventDestroy(e);
  if (ctx->ev_start) cudaEventDestroy(ctx->ev_start);
  if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
  delete ctx;
  return 0;
}

DMNERF_API int dmnerf_set_weights(dmnerf_ctx* ctx, int net, const float* const* params, int n_params, int ins_num, void* stream) {
  DMN_CHECK(ctx != nullptr, "set_weights: ctx is NULL");
  DMN_CHECK(net == 0 || net == 1, "set_weights: net must be 0 (coarse) or 1 (fine), got %d", net);
  DMN_CHECK(n_params == DMNERF_N_PARAMS, "set_weights: expected %d tensors (state_dict order), got %d",
            DMNERF_N_PARAMS, n_params);
  DMN_CHECK(ins_num >= 1 && ins_num <= DMNERF_MAX_INS, "set_weights: ins_num=%d out of range [1,%d]", ins_num,
            DMNERF_MAX_INS);
  NetParams& p = ctx->net[net];
  for (int l = 0; l < N_LAYERS; ++l) {
    DMN_CHECK(params[2 * l] && params[2 * l + 1], "set_weights: parameter %d is NULL", 2 * l);
    p.w[l] = params[2 * l];
    p.b[l] = params[2 * l + 1];
  }
  p.ins_num = ins_num;
  p.bound = true;
  return umma_weights_pack(ctx->packed[net], p, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_posenc(const float* x, int64_t m, int n_freqs, float* out, void* stream) {
  DMN_CHECK(m >= 0, "posenc: negative row count");
  DMN_CHECK(m == 0 || (x && out), "posenc: NULL buffer");
  return launch_posenc(x, m, n_freqs, out, (cudaStream_t)stream);
}

static int mlp_dispatch(dmnerf_ctx* ctx, int net, const float* x, const float* ro, const float* rd, const float* z,
                        int64_t m, int s, float* out, int impl, cudaStream_t st) {
  DMN_CHECK(ctx != nullptr, "mlp: ctx is NULL");
  DMN_CHECK(net == 0 || net == 1, "mlp: net must be 0 or 1");
  DMN_CHECK(m >= 0, "mlp: negative row count");
  DMN_CHECK(impl >= DMNERF_IMPL_AUTO && impl <= DMNERF_IMPL_UMMA, "mlp: unknown impl %d", impl);
  if (m == 0) return 0;
  DMN_CHECK(out != nullptr, "mlp: out is NULL");
  if (impl == DMNERF_IMPL_AUTO) impl = umma_available(ctx->packed[net]) ? DMNERF_IMPL_UMMA : DMNERF_IMPL_SIMT;
  if (impl == DMNERF_IMPL_UMMA)
    return launch_mlp_umma(ctx->packed[net], ctx->net[net], x, ro, rd, z, m, s, out, nullptr, st);
  return launch_mlp_simt(ctx->net[net], x, ro, rd, z, m, s, out, nullptr, st);
}

DMNERF_API int dmnerf_mlp_forward(dmnerf_ctx* ctx, int net, const float* x, int64_t m, float* out, int impl, void* stream) {
  DMN_CHECK(m <= 0 || x != nullptr, "mlp_forward: x is NULL");
  return mlp_dispatch(ctx, net, x, nullptr, nullptr, nullptr, m, 1, out, impl, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_mlp_forward_rays(dmnerf_ctx* ctx, int net, const float* rays_o, const float* rays_d, const float* z,
                            int64_t n, int s, float* out, int impl, void* stream) {
  DMN_CHECK(n >= 0 && s >= 1, "mlp_forward_rays: bad sizes n=%lld s=%d", (long long)n, s);
  DMN_CHECK(n == 0 || (rays_o && rays_d && z), "mlp_forward_rays: NULL input");
  return mlp_dispatch(ctx, net, nullptr, rays_o, rays_d, z, n * s, s, out, impl, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_mlp_forward_points(dmnerf_ctx* ctx, int net, const float* pts, const float* viewdirs, int64_t m, float* out,
                                         int impl, void* stream) {
  DMN_CHECK(ctx != nullptr && (net == 0 || net == 1), "mlp_forward_points: bad ctx / net");
  DMN_CHECK(m >= 0, "mlp_forward_points: negative point count");
  DMN_CHECK(m == 0 || (pts && viewdirs && out), "mlp_forward_points: NULL buffer");
  DMN_CHECK(impl != DMNERF_IMPL_SIMT, "mlp_forward_points: the point query runs on the tensor-core kernel only");
  if (m == 0) return 0;
  DMN_CHECK(umma_available(ctx->packed[net]), "mlp_forward_points: bind the network with dmnerf_set_weights first");
  return launch_mlp_umma(ctx->packed[net], ctx->net[net], nullptr, pts, viewdirs, nullptr, m, 1, out, nullptr, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_composite(const float* raw, const float* z, const float* rays_d, int64_t n, int s, int c, int keep_all_ins,
                     float* rgb, float* weights, float* depth, float* ins, float* acc, void* stream) {
  DMN_CHECK(n >= 0, "composite: negative ray count");
  DMN_CHECK(n == 0 || (raw && z && rays_d), "composite: NULL input");
  return launch_composite(raw, z, rays_d, n, s, c, keep_all_ins, rgb, weights, depth, ins, acc, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_sample_pdf(const float* bins, const float* weights, int64_t n, int n_bins, int n_samples, const float* u,
                      float* out, void* stream) {
  DMN_CHECK(n >= 0, "sample_pdf: negative ray count");
  DMN_CHECK(n == 0 || (bins && weights && out), "sample_pdf: NULL buffer");
  return launch_sample_pdf(bins, weights, n, n_bins, n_samples, u, out, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_sort_concat(const float* a, const float* b, int64_t n, int na, int nb, float* out, void* stream) {
  DMN_CHECK(n >= 0, "sort_concat: negative ray count");
  DMN_CHECK(n == 0 || ((a || na == 0) && (b || nb == 0) && out), "sort_concat: NULL buffer");
  return launch_sort_concat(a, b, n, na, nb, out, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_get_rays(const float* K_host, const float* c2w_host, int H, int W, float* rays_o, float* rays_d, void* stream) {
  DMN_CHECK(K_host && c2w_host && rays_o && rays_d, "get_rays: NULL argument");
  return launch_rays(K_host, c2w_host, H, W, rays_o, rays_d, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_get_rays_at(const float* K_host, const float* c2w_host, int H, int W, const int64_t* pixels, int64_t n,
                                  float* rays_o, float* rays_d, void* stream) {
  DMN_CHECK(K_host && c2w_host && (n == 0 || (pixels && rays_o && rays_d)), "get_rays_at: NULL argument");
  DMN_CHECK(n >= 0, "get_rays_at: negative count");
  return launch_rays_at(K_host, c2w_host, nullptr, 0, H, W, pixels, n, rays_o, rays_d, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_get_rays_at_dev(const float* K_host, const float* c2w_dev, int64_t c2w_row_stride, int H, int W,
                                      const int64_t* pixels, int64_t n, float* rays_o, float* rays_d, void* stream) {
  DMN_CHECK(K_host && c2w_dev && (n == 0 || (pixels && rays_o && rays_d)), "get_rays_at_dev: NULL argument");
  DMN_CHECK(n >= 0 && c2w_row_stride >= 4, "get_rays_at_dev: bad count / row stride");
  return launch_rays_at(K_host, nullptr, c2w_dev, c2w_row_stride, H, W, pixels, n, rays_o, rays_d, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_select_pixels(uint64_t seed, int H, int W, int64_t n, int64_t* pixels, void* stream) {
  DMN_CHECK(n == 0 || pixels, "select_pixels: NULL buffer");
  return launch_select_pixels(seed, H, W, n, pixels, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_hungarian_costs(const float* pred, const int32_t* gt_row, int64_t n, int ins_num, float* cost_ce,
                                      float* cost_siou, float* tp, float* col_sum, float* row_count, void* stream) {
  DMN_CHECK(pred && gt_row && cost_ce && cost_siou && tp && col_sum && row_count, "hungarian_costs: NULL buffer");
  return launch_hungarian_costs(pred, gt_row, n, ins_num, cost_ce, cost_siou, tp, col_sum, row_count, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_ins_loss_backward(const float* pred, const int32_t* gt_row, int64_t n, int ins_num,
                                        const int32_t* row_of_col, int n_valid, const float* tp, const float* col_sum,
                                        const float* row_count, const float* g_losses, float* d_pred, void* stream) {
  DMN_CHECK(n >= 0, "ins_loss_backward: negative ray count");
  DMN_CHECK(n == 0 || (pred && gt_row && row_of_col && tp && col_sum && row_count && g_losses && d_pred),
            "ins_loss_backward: NULL buffer");
  return launch_ins_loss_grad(pred, gt_row, n, ins_num, row_of_col, n_valid, nullptr, tp, col_sum, row_count, g_losses, d_pred,
                              (cudaStream_t)stream);
}

DMNERF_API int dmnerf_ins_label_rows(const int32_t* labels, int64_t n, int ins_num, int32_t* gt_row, int32_t* n_valid, void* stream) {
  DMN_CHECK(labels && gt_row && n_valid, "ins_label_rows: NULL buffer");
  return launch_label_rows(labels, n, ins_num, gt_row, n_valid, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_hungarian_assign(const float* cost_ce, const float* cost_siou, const float* col_sum, const int32_t* n_valid,
                                       int64_t n, int ins_num, int32_t* row_of_col, float* losses, void* stream) {
  DMN_CHECK(cost_ce && cost_siou && col_sum && n_valid && row_of_col && losses, "hungarian_assign: NULL buffer");
  return launch_hungarian_assign(cost_ce, cost_siou, col_sum, n_valid, n, ins_num, row_of_col, losses, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_ins_loss_backward_dev(const float* pred, const int32_t* gt_row, int64_t n, int ins_num,
                                            const int32_t* row_of_col, const int32_t* n_valid, const float* tp, const float* col_sum,
                                            const float* row_count, const float* g_losses, float* d_pred, void* stream) {
  DMN_CHECK(n >= 0, "ins_loss_backward_dev: negative ray count");
  DMN_CHECK(n == 0 || (pred && gt_row && row_of_col && n_valid && tp && col_sum && row_count && g_losses && d_pred),
            "ins_loss_backward_dev: NULL buffer");
  return launch_ins_loss_grad(pred, gt_row, n, ins_num, row_of_col, 0, n_valid, tp, col_sum, row_count, g_losses, d_pred,
                              (cudaStream_t)stream);
}

DMNERF_API int dmnerf_ins_status_take(void) { return ins_status_take(); }

DMNERF_API int dmnerf_stratify(const float* z_in, int64_t z_row_stride, const float* t_rand, int64_t n, int s, float* z_out,
                               void* stream) {
  DMN_CHECK(n >= 0 && s >= 1, "stratify: bad sizes");
  DMN_CHECK(n == 0 || (z_in && z_out), "stratify: NULL buffer");
  DMN_CHECK(z_row_stride == 0 || z_row_stride >= s, "stratify: bad z_row_stride");
  return launch_prep_z(z_in, z_row_stride, t_rand, n, s, z_out, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_hier_sample(const float* z_c, const float* w_c, const float* u, int64_t n, int s, int n_importance,
                                  float* z_fine, void* stream) {
  DMN_CHECK(n >= 0, "hier_sample: negative ray count");
  DMN_CHECK(n == 0 || (z_c && w_c && z_fine), "hier_sample: NULL buffer");
  return launch_hier_sample(z_c, w_c, u, n, s, n_importance, z_fine, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_act_floats_per_sample(void) { return ACT_FLOATS_PER_SAMPLE; }
DMNERF_API int64_t dmnerf_mlp_backward_scratch_floats(int64_t m) { return (int64_t)mlp_backward_scratch_floats(m); }

DMNERF_API int dmnerf_mlp_forward_train(dmnerf_ctx* ctx, int net, const float* x, const float* rays_o, const float* rays_d,
                                        const float* z, int64_t m, int s, float* out, float* acts, int impl, void* stream) {
  DMN_CHECK(ctx != nullptr, "mlp_forward_train: ctx is NULL");
  DMN_CHECK(net == 0 || net == 1, "mlp_forward_train: net must be 0 or 1");
  DMN_CHECK(m >= 0 && s >= 1, "mlp_forward_train: bad sizes");
  if (m == 0) return 0;
  DMN_CHECK(out && acts, "mlp_forward_train: out / acts is NULL");
  DMN_CHECK(impl >= DMNERF_IMPL_AUTO && impl <= DMNERF_IMPL_UMMA, "mlp_forward_train: unknown impl %d", impl);
  if (impl == DMNERF_IMPL_AUTO) impl = umma_available(ctx->packed[net]) ? DMNERF_IMPL_UMMA : DMNERF_IMPL_SIMT;
  ctx->train_feats_missing[net] = (impl == DMNERF_IMPL_UMMA);
  if (impl == DMNERF_IMPL_UMMA)
    return launch_mlp_umma(ctx->packed[net], ctx->net[net], x, rays_o, rays_d, z, m, s, out, acts, (cudaStream_t)stream);
  return launch_mlp_simt(ctx->net[net], x, rays_o, rays_d, z, m, s, out, acts, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_mlp_backward(dmnerf_ctx* ctx, int net, float* acts, const float* d_out, int64_t m, float* const* grads,
                                   float* scratch, int feats_missing, void* stream) {
  DMN_CHECK(ctx != nullptr, "mlp_backward: ctx is NULL");
  DMN_CHECK(net == 0 || net == 1, "mlp_backward: net must be 0 or 1");
  DMN_CHECK(m >= 0 && grads, "mlp_backward: bad arguments");
  DMN_CHECK(m == 0 || (acts && d_out && scratch), "mlp_backward: NULL buffer");
  return launch_mlp_backward(ctx->net[net], &ctx->packed[net], acts, d_out, m, grads, scratch, feats_missing, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_composite_backward(const float* raw, const float* z, const float* rays_d, int64_t n, int s, int c,
                                         int keep_all_ins, const float* g_rgb, const float* g_depth, const float* g_acc,
                                         const float* g_ins, const float* g_weights, float* d_raw, int accumulate, void* stream) {
  DMN_CHECK(n >= 0, "composite_backward: negative ray count");
  DMN_CHECK(n == 0 || (raw && z && rays_d && d_raw), "composite_backward: NULL buffer");
  return launch_composite_backward(raw, z, rays_d, n, s, c, keep_all_ins, g_rgb, g_depth, g_acc, g_ins, g_weights, d_raw,
                                   accumulate, (cudaStream_t)stream);
}

DMNERF_API int64_t dmnerf_penalizer_state_bytes(void) { return (int64_t)penalizer_state_bytes(); }

DMNERF_API int dmnerf_penalizer_forward(const float* raw, const float* z_vals, const float* depth, const float* rays_d, int64_t n,
                                        int s, int c, float tolerance, float deta_w, void* state, float* loss, void* stream) {
  DMN_CHECK(n >= 0, "penalizer_forward: negative ray count");
  DMN_CHECK(state && loss && (n == 0 || (raw && z_vals && depth && rays_d)), "penalizer_forward: NULL buffer");
  DMN_CHECK(deta_w > 0.0f, "penalizer_forward: deta_w must be positive");
  return launch_penalizer_forward(raw, z_vals, depth, rays_d, n, s, c, tolerance, deta_w, state, loss, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_penalizer_backward(const float* raw, const float* z_vals, const float* depth, const float* rays_d, int64_t n,
                                         int s, int c, float tolerance, float deta_w, const void* state, const float* g_loss,
                                         float* d_raw, int accumulate, void* stream) {
  DMN_CHECK(n >= 0, "penalizer_backward: negative ray count");
  DMN_CHECK(state && g_loss && (n == 0 || (raw && z_vals && depth && rays_d && d_raw)), "penalizer_backward: NULL buffer");
  return launch_penalizer_backward(raw, z_vals, depth, rays_d, n, s, c, tolerance, deta_w, state, g_loss, d_raw, accumulate,
                                   (cudaStream_t)stream);
}

DMNERF_API int dmnerf_render_forward(dmnerf_ctx* ctx, const dmnerf_render_io* io, int64_t n, int S, int NI, int flags, int impl,
                          void* stream) {
  DMN_CHECK(ctx && io, "render_forward: NULL ctx/io");
  DMN_CHECK(n >= 0 && S >= 3 && NI >= 2, "render_forward: bad sizes n=%lld S=%d I=%d", (long long)n, S, NI);
  DMN_CHECK(ctx->net[0].bound && ctx->net[1].bound, "render_forward: bind both networks with dmnerf_set_weights first");
  DMN_CHECK(ctx->net[0].ins_num == ctx->net[1].ins_num, "render_forward: coarse/fine ins_num differ");
  if (n == 0) return 0;
  DMN_CHECK(io->rays_o && io->rays_d && io->z_coarse, "render_forward: rays_o / rays_d / z_coarse is NULL");
  const bool perturb = (flags & DMNERF_FLAG_PERTURB) != 0;
  DMN_CHECK(!perturb || (io->t_rand && io->u), "render_forward: PERTURB needs t_rand and u");
  DMN_CHECK(io->z_row_stride == 0 || io->z_row_stride >= S, "render_forward: bad z_row_stride");
  cudaStream_t st = (cudaStream_t)stream;
  const int C = 4 + ctx->net[0].ins_num + 1, F = S + NI;
  const int keep = (flags & DMNERF_FLAG_KEEP_INS) ? 1 : 0;
  DMN_CUDA(cudaSetDevice(ctx->device));

  // ---- fully fused path: one launch, no intermediate tensor in HBM
  const bool can_fuse = impl != DMNERF_IMPL_SIMT && S == 64 && NI == 128 && !io->raw_coarse && !io->raw_fine &&
                        umma_available(ctx->packed[0]) && umma_available(ctx->packed[1]);
  if (can_fuse) {
    const bool prof = ctx->profiling;
    if (prof) DMN_CUDA(cudaEventRecord(ctx->ev[0], st));
    int rc = launch_render_umma(ctx->packed[0], ctx->packed[1], io, n, flags, st);
    if (rc) return rc;
    if (prof) for (int i = 1; i <= DMNERF_N_STAGES; ++i) DMN_CUDA(cudaEventRecord(ctx->ev[i], st));
    ctx->profile_valid = prof;
    ctx->last_fused = true;
    return 0;
  }
  ctx->last_fused = false;

  // scratch for whatever the caller does not want back
  float* z_c = io->z_vals_coarse;
  if (!z_c) { if (ctx->ws_z_c.reserve((size_t)n * S * 4)) return 2; z_c = (float*)ctx->ws_z_c.ptr; }
  float* z_f = io->z_vals_fine;
  if (!z_f) { if (ctx->ws_z_f.reserve((size_t)n * F * 4)) return 2; z_f = (float*)ctx->ws_z_f.ptr; }
  float* w_c = io->weights_coarse;
  if (!w_c) { if (ctx->ws_w_c.reserve((size_t)n * S * 4)) return 2; w_c = (float*)ctx->ws_w_c.ptr; }
  float* raw_c = io->raw_coarse;
  if (!raw_c) { if (ctx->ws_raw_c.reserve((size_t)n * S * C * 4)) return 2; raw_c = (float*)ctx->ws_raw_c.ptr; }
  float* raw_f = io->raw_fine;
  if (!raw_f) { if (ctx->ws_raw_f.reserve((size_t)n * F * C * 4)) return 2; raw_f = (float*)ctx->ws_raw_f.ptr; }

  int rc;
  const bool prof = ctx->profiling;
  int stage = 0;
#define DMN_STAGE_MARK() do { if (prof) DMN_CUDA(cudaEventRecord(ctx->ev[stage++], st)); } while (0)
  DMN_STAGE_MARK();
  // render.py:40-47  coarse depths (+ stratified jitter)
  if ((rc = launch_prep_z(io->z_coarse, io->z_row_stride, perturb ? io->t_rand : nullptr, n, S, z_c, st))) return rc;
  DMN_STAGE_MARK();
  // render.py:49-61  points, embeddings, coarse network
  if ((rc = mlp_dispatch(ctx, 0, nullptr, io->rays_o, io->rays_d, z_c, n * S, S, raw_c, impl, st))) return rc;
  DMN_STAGE_MARK();
  // render.py:63     coarse composite
  if ((rc = launch_composite(raw_c, z_c, io->rays_d, n, S, C, keep, io->rgb_coarse, w_c, io->depth_coarse,
                             io->ins_coarse, io->acc_coarse, st))) return rc;
  DMN_STAGE_MARK();
  // render.py:66-70  importance sampling + merge
  if ((rc = launch_hier_sample(z_c, w_c, perturb ? io->u : nullptr, n, S, NI, z_f, st))) return rc;
  DMN_STAGE_MARK();
  // render.py:71-82  fine network on all S+I depths
  if ((rc = mlp_dispatch(ctx, 1, nullptr, io->rays_o, io->rays_d, z_f, n * F, F, raw_f, impl, st))) return rc;
  DMN_STAGE_MARK();
  // render.py:86     fine composite
  if ((rc = launch_composite(raw_f, z_f, io->rays_d, n, F, C, keep, io->rgb_fine, io->weights_fine, io->depth_fine,
                             io->ins_fine, io->acc_fine, st))) return rc;
  DMN_STAGE_MARK();
#undef DMN_STAGE_MARK
  ctx->profile_valid = prof;
  return 0;
}

DMNERF_API int dmnerf_sync_check(dmnerf_ctx* ctx, void* stream) {
  DMN_CHECK(ctx != nullptr, "sync_check: ctx is NULL");
  DMN_CUDA(cudaSetDevice(ctx->device));
  DMN_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  for (int i = 0; i < 2; ++i) {
    int rc = umma_check_status(ctx->packed[i], (cudaStream_t)stream);
    if (rc) return rc;
  }
  return gemm_tc_check_status((cudaStream_t)stream);
}

DMNERF_API int dmnerf_profile_enable(dmnerf_ctx* ctx, int enable) {
  DMN_CHECK(ctx != nullptr, "profile_enable: ctx is NULL");
  DMN_CUDA(cudaSetDevice(ctx->device));
  if (enable)
    for (cudaEvent_t& e : ctx->ev)
      if (!e) DMN_CUDA(cudaEventCreate(&e));
  ctx->profiling = enable != 0;
  ctx->profile_valid = false;
  return 0;
}

DMNERF_API int dmnerf_profile_read(dmnerf_ctx* ctx, float* ms_out, int n_out) {
  DMN_CHECK(ctx && ms_out, "profile_read: NULL argument");
  DMN_CHECK(n_out >= DMNERF_N_STAGES, "profile_read: need room for %d stages", DMNERF_N_STAGES);
  DMN_CHECK(ctx->profile_valid, "profile_read: no profiled render call recorded");
  DMN_CUDA(cudaEventSynchronize(ctx->ev[DMNERF_N_STAGES]));
  for (int i = 0; i < DMNERF_N_STAGES; ++i) DMN_CUDA(cudaEventElapsedTime(&ms_out[i], ctx->ev[i], ctx->ev[i + 1]));
  return 0;
}

}  // extern "C"

// Host-buffer render: `h` holds HOST pointers for the outputs (and for the inputs unless dev_rays_o / dev_rays_d are given:
// rays that are already resident on the device, e.g. generated there from the camera).
static int render_host_impl(dmnerf_ctx* ctx, const dmnerf_render_io* h, const float* dev_rays_o, const float* dev_rays_d, int64_t n,
                            int S, int NI, int flags, int impl, void* stream) {
  DMN_CHECK(ctx && h, "render_forward_host: NULL ctx/io");
  DMN_CHECK(n >= 0, "render_forward_host: negative ray count");
  if (n == 0) return 0;
  const bool dev_rays = dev_rays_o != nullptr && dev_rays_d != nullptr;
  DMN_CHECK((dev_rays || (h->rays_o && h->rays_d)) && h->z_coarse, "render_forward_host: rays_o / rays_d / z_coarse is NULL");
  DMN_CHECK(ctx->net[0].bound && ctx->net[1].bound, "render_forward_host: bind both networks first");
  cudaStream_t st = (cudaStream_t)stream;
  DMN_CUDA(cudaSetDevice(ctx->device));
  const int ins = ctx->net[0].ins_num, C = 4 + ins + 1, F = S + NI;
  const int n_ins_out = (flags & DMNERF_FLAG_KEEP_INS) ? ins + 1 : ins;
  const bool perturb = (flags & DMNERF_FLAG_PERTURB) != 0;
  const size_t zin = (h->z_row_stride == 0) ? (size_t)S : (size_t)n * h->z_row_stride;

  // ---- inputs: one device arena
  size_t in_floats = (dev_rays ? 0 : (size_t)n * 6) + zin + (perturb ? (size_t)n * (S + NI) : 0);
  if (ctx->host_in.reserve(in_floats * 4)) return 2;
  float* d = (float*)ctx->host_in.ptr;
  dmnerf_render_io io;
  memset(&io, 0, sizeof(io));
  float* p = d;
  float *d_ro = nullptr, *d_rd = nullptr, *d_tr = nullptr, *d_u = nullptr;
  if (dev_rays) {
    io.rays_o = dev_rays_o; io.rays_d = dev_rays_d;
  } else {
    d_ro = p; io.rays_o = p; p += n * 3;
    d_rd = p; io.rays_d = p; p += n * 3;
  }
  float* d_z = p; io.z_coarse = p; p += zin;
  io.z_row_stride = h->z_row_stride;
  if (perturb) {
    DMN_CHECK(h->t_rand && h->u, "render_forward_host: PERTURB needs t_rand and u");
    d_tr = p; io.t_rand = p; p += n * S;
    d_u = p; io.u = p; p += n * NI;
  }
  // ---- outputs: one device arena, carved for every non-NULL host output
  struct Out { float* dmnerf_render_io::* hp; size_t per_ray; };
  const Out outs[] = {
      {&dmnerf_render_io::rgb_coarse, 3}, {&dmnerf_render_io::rgb_fine, 3},
      {&dmnerf_render_io::depth_coarse, 1}, {&dmnerf_render_io::depth_fine, 1},
      {&dmnerf_render_io::acc_coarse, 1}, {&dmnerf_render_io::acc_fine, 1},
      {&dmnerf_render_io::ins_coarse, (size_t)n_ins_out}, {&dmnerf_render_io::ins_fine, (size_t)n_ins_out},
      {&dmnerf_render_io::z_vals_coarse, (size_t)S}, {&dmnerf_render_io::z_vals_fine, (size_t)F},
      {&dmnerf_render_io::weights_coarse, (size_t)S}, {&dmnerf_render_io::weights_fine, (size_t)F},
      {&dmnerf_render_io::raw_coarse, (size_t)S * C}, {&dmnerf_render_io::raw_fine, (size_t)F * C},
  };
  size_t out_floats = 0;
  for (const Out& o : outs) if (h->*(o.hp)) out_floats += (size_t)n * o.per_ray;
  if (ctx->host_out.reserve(out_floats * 4 + 16)) return 2;
  float* q = (float*)ctx->host_out.ptr;
  for (const Out& o : outs) if (h->*(o.hp)) { io.*(o.hp) = q; q += (size_t)n * o.per_ray; }

  // Copies of rows [r0, r1) of the batch.  Every ray is rendered independently of its neighbours (the rows of a tile never
  // mix), so rendering a large batch in parts gives the same bits as one launch.
  auto copy_in = [&](int64_t r0, int64_t r1, cudaStream_t cs) -> int {
    const size_t cnt = (size_t)(r1 - r0);
    if (!dev_rays) {
      DMN_CUDA(cudaMemcpyAsync(d_ro + r0 * 3, h->rays_o + r0 * 3, cnt * 12, cudaMemcpyHostToDevice, cs));
      DMN_CUDA(cudaMemcpyAsync(d_rd + r0 * 3, h->rays_d + r0 * 3, cnt * 12, cudaMemcpyHostToDevice, cs));
    }
    if (h->z_row_stride != 0)
      DMN_CUDA(cudaMemcpyAsync(d_z + r0 * h->z_row_stride, h->z_coarse + r0 * h->z_row_stride, cnt * h->z_row_stride * 4,
                               cudaMemcpyHostToDevice, cs));
    if (perturb) {
      DMN_CUDA(cudaMemcpyAsync(d_tr + r0 * S, h->t_rand + r0 * S, cnt * S * 4, cudaMemcpyHostToDevice, cs));
      DMN_CUDA(cudaMemcpyAsync(d_u + r0 * NI, h->u + r0 * NI, cnt * NI * 4, cudaMemcpyHostToDevice, cs));
    }
    return 0;
  };
  auto copy_out = [&](int64_t r0, int64_t r1, cudaStream_t cs) -> int {
    for (const Out& o : outs)
      if (h->*(o.hp))
        DMN_CUDA(cudaMemcpyAsync(h->*(o.hp) + r0 * o.per_ray, io.*(o.hp) + r0 * o.per_ray, (size_t)(r1 - r0) * o.per_ray * 4,
                                 cudaMemcpyDeviceToHost, cs));
    return 0;
  };
  auto part_io = [&](int64_t r0) {
    dmnerf_render_io pi = io;
    if (pi.rays_o) { pi.rays_o += r0 * 3; pi.rays_d += r0 * 3; }
    if (pi.z_row_stride != 0) pi.z_coarse += r0 * pi.z_row_stride;
    if (pi.t_rand) pi.t_rand += r0 * S;
    if (pi.u) pi.u += r0 * NI;
    for (const Out& o : outs) if (pi.*(o.hp)) pi.*(o.hp) += r0 * o.per_ray;
    return pi;
  };
  if (h->z_row_stride == 0) DMN_CUDA(cudaMemcpyAsync(d_z, h->z_coarse, zin * 4, cudaMemcpyHostToDevice, st));   // the shared depth row

  const bool parts = n >= HOST_PART_MIN_RAYS && !ctx->profiling;
  if (!parts) {
    if (copy_in(0, n, st)) return 1;
    int rc = dmnerf_render_forward(ctx, &io, n, S, NI, flags, impl, stream);
    if (rc) return rc;
    if (copy_out(0, n, st)) return 1;
    return dmnerf_sync_check(ctx, stream);
  }
  // Large batch: HOST_PARTS launches on the caller's stream; the inputs of part i+1 and the maps of part i-1 travel on a second
  // stream while part i is rendered, so that only the first upload and the last download are not hidden behind kernels.
  if (!ctx->copy_stream) {
    DMN_CUDA(cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
    for (int i = 0; i < HOST_PARTS; ++i) {
      DMN_CUDA(cudaEventCreateWithFlags(&ctx->ev_in[i], cudaEventDisableTiming));
      DMN_CUDA(cudaEventCreateWithFlags(&ctx->ev_done[i], cudaEventDisableTiming));
    }
    DMN_CUDA(cudaEventCreateWithFlags(&ctx->ev_start, cudaEventDisableTiming));
  }
  cudaStream_t cs = ctx->copy_stream;
  int64_t edge[HOST_PARTS + 1];
  for (int i = 0; i <= HOST_PARTS; ++i) edge[i] = ((n * i / HOST_PARTS) + 1) & ~(int64_t)1;      // even boundaries: whole ray pairs
  edge[0] = 0; edge[HOST_PARTS] = n;
  DMN_CUDA(cudaEventRecord(ctx->ev_start, st));                   // the copy stream starts after everything already queued on st
  DMN_CUDA(cudaStreamWaitEvent(cs, ctx->ev_start, 0));
  if (copy_in(edge[0], edge[1], st)) return 1;
  for (int i = 1; i < HOST_PARTS; ++i) {
    if (copy_in(edge[i], edge[i + 1], cs)) return 1;
    DMN_CUDA(cudaEventRecord(ctx->ev_in[i], cs));
  }
  int rc = 0;
  for (int i = 0; i < HOST_PARTS && !rc; ++i) {
    if (i > 0) DMN_CUDA(cudaStreamWaitEvent(st, ctx->ev_in[i], 0));
    const dmnerf_render_io pi = part_io(edge[i]);
    rc = dmnerf_render_forward(ctx, &pi, edge[i + 1] - edge[i], S, NI, flags, impl, stream);
    if (rc) break;
    DMN_CUDA(cudaEventRecord(ctx->ev_done[i], st));
    DMN_CUDA(cudaStreamWaitEvent(cs, ctx->ev_done[i], 0));
    if (copy_out(edge[i], edge[i + 1], cs)) { rc = 1; break; }
  }
  const cudaError_t ce = cudaStreamSynchronize(cs);               // also on the error path: nothing of this call stays in flight
  if (rc) { cudaStreamSynchronize(st); return rc; }
  DMN_CUDA(ce);
  return dmnerf_sync_check(ctx, stream);
}

extern "C" {

DMNERF_API int dmnerf_render_forward_host(dmnerf_ctx* ctx, const dmnerf_render_io* h, int64_t n, int S, int NI, int flags,
                               int impl, void* stream) {
  return render_host_impl(ctx, h, nullptr, nullptr, n, S, NI, flags, impl, stream);
}

DMNERF_API int dmnerf_render_frame_host(dmnerf_ctx* ctx, const float* K_host, const float* c2w_host, int H, int W, float near_z,
                                        float far_z, int64_t ray_begin, int64_t ray_count, int n_coarse, int n_importance,
                                        int flags, int impl, const dmnerf_render_io* out_host, void* stream) {
  DMN_CHECK(ctx && K_host && c2w_host && out_host, "render_frame_host: NULL argument");
  DMN_CHECK(H > 0 && W > 0 && n_coarse >= 3 && n_coarse <= 4096, "render_frame_host: bad sizes H=%d W=%d S=%d", H, W, n_coarse);
  DMN_CHECK(ray_begin >= 0 && ray_count >= 0 && ray_begin + ray_count <= (int64_t)H * W,
            "render_frame_host: pixel range [%lld, +%lld) outside the %dx%d frame", (long long)ray_begin, (long long)ray_count, H, W);
  DMN_CHECK(!(flags & DMNERF_FLAG_PERTURB), "render_frame_host: the frame driver is the deterministic test-time path");
  if (ray_count == 0) return 0;
  DMN_CUDA(cudaSetDevice(ctx->device));
  // rays of the whole frame on the device (helpers.py:50-61; tester.py:59-61), the range asked for is rendered
  if (ctx->frame_rays.reserve((size_t)H * W * 6 * sizeof(float))) return 2;
  float* ro = (float*)ctx->frame_rays.ptr;
  float* rd = ro + (size_t)H * W * 3;
  int rc = dmnerf_get_rays(K_host, c2w_host, H, W, ro, rd, stream);
  if (rc) return rc;
  // z_val_sample (helpers.py:114-119): near + linspace(0, 1, S) * (far - near), torch.linspace's symmetric fp32 evaluation
  std::vector<float> z((size_t)n_coarse);
  const float step = 1.0f / (float)(n_coarse - 1), span = far_z - near_z;
  for (int i = 0; i < n_coarse; ++i) {
    const float t = (i < n_coarse / 2) ? step * (float)i : fmaf(-step, (float)(n_coarse - 1 - i), 1.0f);
    z[i] = near_z + t * span;
  }
  dmnerf_render_io h = *out_host;
  h.rays_o = nullptr; h.rays_d = nullptr; h.t_rand = nullptr; h.u = nullptr;
  h.z_coarse = z.data(); h.z_row_stride = 0;
  return render_host_impl(ctx, &h, ro + ray_begin * 3, rd + ray_begin * 3, ray_count, n_coarse, n_importance, flags, impl, stream);
}

// ---- mesh extraction (tools/mesh_generator.py mesh_main) ------------------------------------------------------------------

DMNERF_API int dmnerf_mesh_grid_points(const double* transform_host, const double* extents_host, int dim, int64_t begin, int64_t count,
                                       float* pts, void* stream) {
  DMN_CHECK(transform_host && extents_host && (count == 0 || pts), "mesh_grid_points: NULL argument");
  return launch_grid_points(transform_host, extents_host, dim, begin, count, pts, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_mesh_occupancy(dmnerf_ctx* ctx, int net, const double* transform_host, const double* extents_host, int dim,
                                     float voxel, int64_t slab, float* occ, void* stream) {
  DMN_CHECK(ctx && (net == 0 || net == 1), "mesh_occupancy: bad ctx / net");
  DMN_CHECK(transform_host && extents_host && occ, "mesh_occupancy: NULL argument");
  DMN_CHECK(dim >= 2 && dim <= 2048, "mesh_occupancy: dim %d out of range [2, 2048]", dim);
  DMN_CHECK(umma_available(ctx->packed[net]), "mesh_occupancy: bind the network with dmnerf_set_weights first");
  cudaStream_t st = (cudaStream_t)stream;
  DMN_CUDA(cudaSetDevice(ctx->device));
  const int64_t n = (int64_t)dim * dim * dim;
  if (slab <= 0) slab = (int64_t)1 << 20;
  if (slab > n) slab = n;
  const int C = 4 + ctx->net[net].ins_num + 1;
  if (ctx->mesh_pts.reserve((size_t)slab * 6 * sizeof(float)) || ctx->mesh_raw.reserve((size_t)slab * C * sizeof(float))) return 2;
  float* pts = (float*)ctx->mesh_pts.ptr;
  float* dirs = pts + slab * 3;                                   // mesh_generator.py:42: zero view directions
  float* raw = (float*)ctx->mesh_raw.ptr;
  DMN_CUDA(cudaMemsetAsync(dirs, 0, (size_t)slab * 3 * sizeof(float), st));
  // slab by slab: the [dim^3, C] network output of the original never exists, only [slab, C]
  for (int64_t b = 0; b < n; b += slab) {
    const int64_t cnt = n - b < slab ? n - b : slab;
    int rc = launch_grid_points(transform_host, extents_host, dim, b, cnt, pts, st);
    if (!rc) rc = launch_mlp_umma(ctx->packed[net], ctx->net[net], nullptr, pts, dirs, nullptr, cnt, 1, raw, nullptr, st);
    if (!rc) rc = launch_occupancy(raw, cnt, C, voxel, occ + b, st);
    if (rc) return rc;
  }
  return 0;
}

DMNERF_API int dmnerf_mesh_mc_count(dmnerf_ctx* ctx, const float* grid, int nx, int ny, int nz, float level, int64_t* counts_host,
                                    void* stream) {
  DMN_CHECK(ctx && grid && counts_host, "mesh_mc_count: NULL argument");
  DMN_CUDA(cudaSetDevice(ctx->device));
  return mc_count(&ctx->mesh, grid, nx, ny, nz, level, counts_host, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_mesh_mc_emit(dmnerf_ctx* ctx, const float* grid, int nx, int ny, int nz, float level, float* verts, int32_t* tris,
                                   void* stream) {
  DMN_CHECK(ctx && grid, "mesh_mc_emit: NULL argument");
  DMN_CUDA(cudaSetDevice(ctx->device));
  return mc_emit(ctx->mesh, grid, nx, ny, nz, level, verts, tris, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_mesh_to_scene(const float* verts, int64_t n, const double* transform_host, const double* extents_host, int dim,
                                    float* out, void* stream) {
  DMN_CHECK(n >= 0 && transform_host && extents_host && (n == 0 || (verts && out)), "mesh_to_scene: bad argument");
  return launch_to_scene(verts, n, transform_host, extents_host, dim, out, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_mesh_normals(dmnerf_ctx* ctx, const float* verts, int64_t nv, const int32_t* tris, int64_t nt, float* normals,
                                   void* stream) {
  DMN_CHECK(ctx && (nv == 0 || (verts && normals)) && (nt == 0 || tris), "mesh_normals: NULL argument");
  DMN_CUDA(cudaSetDevice(ctx->device));
  return mesh_normals(&ctx->mesh, verts, nv, tris, nt, normals, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_mesh_clusters(dmnerf_ctx* ctx, const int32_t* tris, int64_t nt, int64_t nv, int32_t* cluster, int32_t* cluster_size,
                                    void* stream) {
  DMN_CHECK(ctx && (nt == 0 || (tris && cluster && cluster_size)), "mesh_clusters: NULL argument");
  DMN_CUDA(cudaSetDevice(ctx->device));
  return mesh_clusters(&ctx->mesh, tris, nt, nv, cluster, cluster_size, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_mesh_clean(dmnerf_ctx* ctx, const float* verts, const float* normals, int64_t nv, const int32_t* tris, int64_t nt,
                                 const int32_t* cluster_size, int min_cluster, float* out_verts, float* out_normals, int32_t* out_tris,
                                 int64_t* counts_host, void* stream) {
  DMN_CHECK(ctx && counts_host, "mesh_clean: NULL argument");
  DMN_CHECK(nv == 0 || (verts && out_verts && (!normals == !out_normals)), "mesh_clean: NULL vertex buffer");
  DMN_CHECK(nt == 0 || (tris && cluster_size && out_tris), "mesh_clean: NULL triangle buffer");
  DMN_CUDA(cudaSetDevice(ctx->device));
  return mesh_clean(&ctx->mesh, verts, normals, nv, tris, nt, cluster_size, min_cluster, out_verts, out_normals, out_tris, counts_host,
                    (cudaStream_t)stream);
}

DMNERF_API int dmnerf_mesh_label_rays(const float* verts, const float* normals, int64_t n, float near_z, float* rays_o, float* rays_d,
                                      void* stream) {
  DMN_CHECK(n >= 0 && (n == 0 || (verts && normals && rays_o && rays_d)), "mesh_label_rays: bad argument");
  return launch_label_rays(verts, normals, n, near_z, rays_o, rays_d, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_argmax_rows(const float* x, int64_t n, int c, int64_t* out, void* stream) {
  DMN_CHECK(n >= 0 && c >= 1 && (n == 0 || (x && out)), "argmax_rows: bad argument");
  return launch_argmax_rows(x, n, c, out, (cudaStream_t)stream);
}

}  // extern "C"
