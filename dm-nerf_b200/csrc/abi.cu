// extern "C" boundary of libdmnerf_b200.so: context, weight binding, stage entry points and the
// whole-pipeline render call.  See include/dmnerf_b200.h for the contract of every symbol.
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "network.cuh"

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

// An entry point's object selection: keep_host (4 host words) -> m, or every label when keep_host is NULL.  Only labels
// 0 .. n_labels - 1 may be set.
static int object_mask(const uint32_t* keep_host, int n_labels, ObjMask& m, const char* who) {
  m = ObjMask{{~0u, ~0u, ~0u, ~0u}};
  if (!keep_host) return 0;
  for (int b = n_labels; b < 128; ++b)
    DMN_CHECK(!((keep_host[b >> 5] >> (b & 31)) & 1u), "%s: object mask keeps label %d, outside [0, %d]", who, b, n_labels - 1);
  for (int i = 0; i < 4; ++i) m.w[i] = keep_host[i];
  return 0;
}

}  // namespace dmnerf

using namespace dmnerf;

constexpr int HOST_PARTS = 4;              // a *_host call on >= HOST_PART_MIN_RAYS rays is rendered in this many parts
constexpr int64_t HOST_PART_MIN_RAYS = 131072;

struct dmnerf_ctx {
  int device = 0;
  Network net[2];                 // 0: coarse, 1: fine (network.cuh)
  DeviceBuffer ws_raw_c, ws_raw_f, ws_z_c, ws_z_f, ws_w_c, ws_w_f;
  DeviceBuffer host_in, host_out; // device staging for the *_host entry point
  DeviceBuffer frame_rays;        // rays of the frame being rendered by dmnerf_render_frame_host
  DeviceBuffer mesh_pts, mesh_raw;   // one slab of the occupancy sweep: points + zero view directions, network output
  DeviceBuffer gemm_wimage, gemm_partial;   // dmnerf_mlp_backward: scratch of the tensor-core GEMMs (gemm_umma.cu)
  MeshState mesh;                 // buffers of the other mesh entry points (mesh.cu)
  InventoryState inventory;       // buffers of the object-inventory entry points (inventory.cu)
  ComponentsState components;     // buffers of the connected-component entry points (components.cu)
  DeviceBuffer region_tmp;        // dmnerf_region_dilate: the second buffer of a multi-step dilation
  // the appearance table of the render call (scene_edit), sized for DMNERF_MAX_INS + 1 rows so that it is never reallocated
  DeviceBuffer appearance_buf;
  bool profiling = false;
  bool profile_valid = false;
  cudaEvent_t ev[DMNERF_N_STAGES + 1] = {};
  // *_host entry points: second stream + events so that the copies of one part of a large batch overlap the kernels of the next
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_in[HOST_PARTS] = {}, ev_done[HOST_PARTS] = {}, ev_start = nullptr;
};

// The precondition of every entry point that runs a network: slot `net` bound with dmnerf_set_weights (and so packed).
static int bound_net(const dmnerf_ctx* ctx, int net, const char* who) {
  DMN_CHECK(ctx != nullptr, "%s: ctx is NULL", who);
  DMN_CHECK(net == 0 || net == 1, "%s: net must be 0 (coarse) or 1 (fine), got %d", who, net);
  DMN_CHECK(ctx->net[net].bound, "%s: bind the network with dmnerf_set_weights first", who);
  return 0;
}

// The precondition of every render entry point: the coarse / fine pair bound with one ins_num.
static int bound_pair(const dmnerf_ctx* ctx, const char* who) {
  DMN_CHECK(ctx != nullptr, "%s: ctx is NULL", who);
  DMN_CHECK(ctx->net[0].bound && ctx->net[1].bound, "%s: bind both networks with dmnerf_set_weights first", who);
  DMN_CHECK(ctx->net[0].p.ins_num == ctx->net[1].p.ins_num, "%s: coarse/fine ins_num differ", who);
  return 0;
}

// The flags the render entry points take.
constexpr int RENDER_FLAGS = DMNERF_FLAG_PERTURB | DMNERF_FLAG_WANT_RAW | DMNERF_FLAG_KEEP_INS;

// The scene edit of a render call, checked against the coarse / fine pair (bound_pair): in (NULL, or all three members NULL: no
// edit) -> e and edit = &e, or edit = NULL for the unselected kernels.  The appearance table is copied on `st`
// into the context's staging buffer.  Without a selection every label is kept (object_mask).
static int scene_edit(dmnerf_ctx* ctx, const dmnerf_edit* in, cudaStream_t st, Edit& e, const Edit*& edit, const char* who) {
  edit = nullptr;
  if (!in || (!in->keep && !in->region && !in->appearance)) return 0;
  const int n_labels = ctx->net[0].p.ins_num + 1;
  if (object_mask(in->keep, n_labels, e.keep, who)) return 1;
  e.region = Region{};
  if (in->region) {
    if (region_from_abi(*in->region, e.region, who)) return 1;
    for (int b = n_labels; b < 128; ++b)
      DMN_CHECK(!obj_kept(e.region.applies, b), "%s: region applies to label %d, outside [0, %d]", who, b, n_labels - 1);
  }
  e.appearance = nullptr;
  if (in->appearance) {
    const int rows = in->appearance_labels;
    DMN_CHECK(rows >= 2 && rows <= DMNERF_MAX_INS + 1, "%s: an appearance of %d labels outside [2, %d]", who, rows,
              DMNERF_MAX_INS + 1);
    DMN_CHECK(rows == n_labels, "%s: the appearance has %d rows for %d labels (ins_num + 1)", who, rows, n_labels);
    for (int l = 0; l < rows; ++l) {
      const float* row = in->appearance + (size_t)l * APPEARANCE_ROW;
      for (int i = 0; i < APPEARANCE_ROW; ++i)
        DMN_CHECK(std::isfinite(row[i]), "%s: appearance entry %d of label %d is not finite", who, i, l);
      DMN_CHECK(row[12] >= 0.0f, "%s: label %d has a negative density scale %g", who, l, (double)row[12]);
    }
    DMN_CUDA(cudaSetDevice(ctx->device));
    float* d;
    if (ctx->appearance_buf.get((size_t)(DMNERF_MAX_INS + 1) * APPEARANCE_ROW, &d)) return 2;
    DMN_CUDA(cudaMemcpyAsync(d, in->appearance, (size_t)rows * APPEARANCE_ROW * sizeof(float), cudaMemcpyHostToDevice, st));
    e.appearance = d;
  }
  edit = &e;
  return 0;
}

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
  DMN_CHECK(params != nullptr, "set_weights: params is NULL");
  for (int i = 0; i < DMNERF_N_PARAMS; ++i) DMN_CHECK(params[i], "set_weights: parameter %d is NULL", i);
  NetParams p;
  for (int l = 0; l < N_LAYERS; ++l) {
    p.w[l] = params[2 * l];
    p.b[l] = params[2 * l + 1];
  }
  p.ins_num = ins_num;
  return ctx->net[net].bind(p, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_posenc(const float* x, int64_t m, int n_freqs, float* out, void* stream) {
  DMN_CHECK(m >= 0, "posenc: negative row count");
  DMN_CHECK(m == 0 || (x && out), "posenc: NULL buffer");
  return launch_posenc(x, m, n_freqs, out, (cudaStream_t)stream);
}

// An fp16 call on caller buffers returns only after its range verdict: synchronise and report (never silent inf / NaN maps).
// A call that failed before its verdict still drains its kernels and drops their verdict: their results are not returned.
static int f16_verdict(dmnerf_ctx* ctx, int rc, int impl, void* stream) {
  if (impl != DMNERF_IMPL_UMMA_F16) return rc;
  if (rc) {
    cudaStreamSynchronize((cudaStream_t)stream);
    for (const Network& n : ctx->net) n.take_f16_range();
    return rc;
  }
  return dmnerf_sync_check(ctx, stream);
}

// The network a call on the bound slots net0 .. net1 runs: impl range-checked, DMNERF_IMPL_AUTO resolved to the tensor-core
// kernel (a bound slot always has its image), and for DMNERF_IMPL_UMMA_F16 every slot's fp16 image packed.
static int resolve_impl(dmnerf_ctx* ctx, int& impl, int net0, int net1, cudaStream_t st, const char* who) {
  DMN_CHECK(impl >= DMNERF_IMPL_AUTO && impl <= DMNERF_IMPL_UMMA_F16, "%s: unknown impl %d", who, impl);
  if (impl == DMNERF_IMPL_AUTO) impl = DMNERF_IMPL_UMMA;
  for (int net = net0; impl == DMNERF_IMPL_UMMA_F16 && net <= net1; ++net)
    if (ctx->net[net].pack_f16(st)) return 1;
  return 0;
}

// The network of the bound slot `net` on m rows.
static int mlp_dispatch(dmnerf_ctx* ctx, int net, const float* x, const float* ro, const float* rd, const float* z,
                        int64_t m, int s, float* out, int impl, cudaStream_t st) {
  DMN_CHECK(m >= 0, "mlp: negative row count");
  if (m == 0) return 0;
  DMN_CHECK(out != nullptr, "mlp: out is NULL");
  if (resolve_impl(ctx, impl, net, net, st, "mlp")) return 1;
  if (impl == DMNERF_IMPL_SIMT) return launch_mlp_simt(ctx->net[net].p, x, ro, rd, z, m, s, out, nullptr, st);
  return launch_mlp_tc(ctx->net[net], x, ro, rd, z, m, s, out, nullptr, st, impl == DMNERF_IMPL_UMMA_F16);
}

DMNERF_API int dmnerf_mlp_forward(dmnerf_ctx* ctx, int net, const float* x, int64_t m, float* out, int impl, void* stream) {
  if (bound_net(ctx, net, "mlp_forward")) return 1;
  DMN_CHECK(m <= 0 || x != nullptr, "mlp_forward: x is NULL");
  return f16_verdict(ctx, mlp_dispatch(ctx, net, x, nullptr, nullptr, nullptr, m, 1, out, impl, (cudaStream_t)stream), impl, stream);
}

DMNERF_API int dmnerf_mlp_forward_rays(dmnerf_ctx* ctx, int net, const float* rays_o, const float* rays_d, const float* z,
                            int64_t n, int s, float* out, int impl, void* stream) {
  if (bound_net(ctx, net, "mlp_forward_rays")) return 1;
  DMN_CHECK(n >= 0 && s >= 1, "mlp_forward_rays: bad sizes n=%lld s=%d", (long long)n, s);
  DMN_CHECK(n == 0 || (rays_o && rays_d && z), "mlp_forward_rays: NULL input");
  return f16_verdict(ctx, mlp_dispatch(ctx, net, nullptr, rays_o, rays_d, z, n * s, s, out, impl, (cudaStream_t)stream), impl,
                     stream);
}

DMNERF_API int dmnerf_mlp_forward_points(dmnerf_ctx* ctx, int net, const float* pts, const float* viewdirs, int64_t m, float* out,
                                         int impl, void* stream) {
  if (bound_net(ctx, net, "mlp_forward_points")) return 1;
  DMN_CHECK(m >= 0, "mlp_forward_points: negative point count");
  DMN_CHECK(m == 0 || (pts && viewdirs && out), "mlp_forward_points: NULL buffer");
  DMN_CHECK(impl != DMNERF_IMPL_SIMT, "mlp_forward_points: the point query runs on the tensor-core kernel only");
  if (m == 0) return 0;
  if (resolve_impl(ctx, impl, net, net, (cudaStream_t)stream, "mlp_forward_points")) return 1;
  return f16_verdict(ctx, launch_mlp_tc(ctx->net[net], nullptr, pts, viewdirs, nullptr, m, 1, out, nullptr, (cudaStream_t)stream,
                                        impl == DMNERF_IMPL_UMMA_F16), impl, stream);
}

DMNERF_API int dmnerf_composite(const float* raw, const float* z, const float* rays_d, int64_t n, int s, int c, int keep_all_ins,
                                const uint32_t* keep_host, float* rgb, float* weights, float* depth, float* ins, float* acc,
                                void* stream) {
  DMN_CHECK(n >= 0, "composite: negative ray count");
  DMN_CHECK(n == 0 || (raw && z && rays_d), "composite: NULL input");
  DMN_CHECK(c >= 5 && c <= 4 + DMNERF_MAX_INS + 1, "composite: channels=%d out of range", c);
  Edit e = {};
  if (object_mask(keep_host, c - 4, e.keep, "composite")) return 1;
  return launch_composite(raw, z, rays_d, n, s, c, keep_all_ins, rgb, weights, depth, ins, acc, (cudaStream_t)stream,
                          keep_host ? &e : nullptr);
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

DMNERF_API int dmnerf_ins_loss_backward(const float* pred, const int32_t* gt_row, int64_t n, int64_t n_global, int ins_num,
                                        const int32_t* row_of_col, const int32_t* n_valid, const float* tp, const float* col_sum,
                                        const float* row_count, const float* g_losses, float* d_pred, void* stream) {
  DMN_CHECK(n >= 0, "ins_loss_backward: negative ray count");
  DMN_CHECK(n == 0 || (pred && gt_row && row_of_col && n_valid && tp && col_sum && row_count && g_losses && d_pred),
            "ins_loss_backward: NULL buffer");
  return launch_ins_loss_grad(pred, gt_row, n, n_global, ins_num, row_of_col, n_valid, tp, col_sum, row_count, g_losses, d_pred,
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

DMNERF_API int dmnerf_ins_label_bitmap(const int32_t* labels, int64_t n, uint32_t* bitmap, void* stream) {
  DMN_CHECK(bitmap && (n == 0 || labels), "ins_label_bitmap: NULL buffer");
  return launch_label_bitmap(labels, n, bitmap, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_ins_label_rows_merged(const uint32_t* bitmaps, int world, const int32_t* labels, int64_t n, int ins_num,
                                            int32_t* gt_row, int32_t* n_valid, void* stream) {
  DMN_CHECK(bitmaps && n_valid && (n == 0 || (labels && gt_row)), "ins_label_rows_merged: NULL buffer");
  return launch_label_rows_merged(bitmaps, world, labels, n, ins_num, gt_row, n_valid, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_hungarian_partials(const float* pred, const int32_t* gt_row, int64_t n, int ins_num, double* partials,
                                         void* stream) {
  DMN_CHECK(partials && (n == 0 || (pred && gt_row)), "hungarian_partials: NULL buffer");
  return launch_hungarian_partials(pred, gt_row, n, ins_num, partials, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_hungarian_costs_merged(const double* partials, int world, int64_t n_global, int ins_num, float* cost_ce,
                                             float* cost_siou, float* tp, float* col_sum, float* row_count, void* stream) {
  DMN_CHECK(partials && cost_ce && cost_siou && tp && col_sum && row_count, "hungarian_costs_merged: NULL buffer");
  return launch_hungarian_costs_merged(partials, world, n_global, ins_num, cost_ce, cost_siou, tp, col_sum, row_count,
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
  if (bound_net(ctx, net, "mlp_forward_train")) return 1;
  DMN_CHECK(m >= 0 && s >= 1, "mlp_forward_train: bad sizes");
  if (m == 0) return 0;
  DMN_CHECK(out && acts, "mlp_forward_train: out / acts is NULL");
  DMN_CHECK(impl != DMNERF_IMPL_UMMA_F16, "mlp_forward_train: DMNERF_IMPL_UMMA_F16 is inference-only; training runs the exact "
            "network (DMNERF_IMPL_UMMA or DMNERF_IMPL_SIMT)");
  if (resolve_impl(ctx, impl, net, net, (cudaStream_t)stream, "mlp_forward_train")) return 1;
  if (impl == DMNERF_IMPL_SIMT) return launch_mlp_simt(ctx->net[net].p, x, rays_o, rays_d, z, m, s, out, acts, (cudaStream_t)stream);
  return launch_mlp_tc(ctx->net[net], x, rays_o, rays_d, z, m, s, out, acts, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_mlp_backward(dmnerf_ctx* ctx, int net, float* acts, const float* d_out, int64_t m, float* const* grads,
                                   float* scratch, int flags, void* stream) {
  if (bound_net(ctx, net, "mlp_backward")) return 1;
  DMN_CHECK(m >= 0 && grads, "mlp_backward: bad arguments");
  DMN_CHECK(m == 0 || (acts && d_out && scratch), "mlp_backward: NULL buffer");
  return launch_mlp_backward(ctx->net[net], acts, d_out, m, grads, scratch, flags, ctx->gemm_wimage, ctx->gemm_partial,
                             (cudaStream_t)stream);
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

DMNERF_API int64_t dmnerf_penalizer_partials_bytes(int64_t n, int s, int c) {
  return (n < 0 || s < 1) ? -1 : (int64_t)penalizer_partials_bytes(n, s, c);
}

DMNERF_API int dmnerf_penalizer_merge(const void* states, int world, int c, void* state, float* loss, void* stream) {
  DMN_CHECK(states && state && loss, "penalizer_merge: NULL buffer");
  return launch_penalizer_merge(states, world, c, state, loss, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_penalizer_forward(const float* raw, const float* z_vals, const float* depth, const float* rays_d, int64_t n,
                                        int s, int c, float tolerance, float deta_w, void* partials, float* loss, void* stream) {
  DMN_CHECK(n >= 0, "penalizer_forward: negative ray count");
  DMN_CHECK(partials && loss && (n == 0 || (raw && z_vals && depth && rays_d)), "penalizer_forward: NULL buffer");
  DMN_CHECK(deta_w > 0.0f, "penalizer_forward: deta_w must be positive");
  return launch_penalizer_forward(raw, z_vals, depth, rays_d, n, s, c, tolerance, deta_w, partials, loss, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_penalizer_backward(const float* raw, const float* z_vals, const float* depth, const float* rays_d, int64_t n,
                                         int s, int c, float tolerance, float deta_w, const void* state, const float* g_loss,
                                         float* d_raw, int accumulate, void* stream) {
  DMN_CHECK(n >= 0, "penalizer_backward: negative ray count");
  DMN_CHECK(state && g_loss && (n == 0 || (raw && z_vals && depth && rays_d && d_raw)), "penalizer_backward: NULL buffer");
  return launch_penalizer_backward(raw, z_vals, depth, rays_d, n, s, c, tolerance, deta_w, state, g_loss, d_raw, accumulate,
                                   (cudaStream_t)stream);
}

}  // extern "C"

// dm_nerf() on device buffers with the bound pair (bound_pair); edit: the checked scene edit, or NULL for none (the
// unselected kernels)
static int render_forward_impl(dmnerf_ctx* ctx, const dmnerf_render_io* io, int64_t n, int S, int NI, int flags, int impl,
                               const Edit* edit, void* stream) {
  DMN_CHECK(io, "render_forward: io is NULL");
  DMN_CHECK(n >= 0 && S >= 3 && NI >= 2, "render_forward: bad sizes n=%lld S=%d I=%d", (long long)n, S, NI);
  if (n == 0) return 0;
  DMN_CHECK(io->rays_o && io->rays_d && io->z_coarse, "render_forward: rays_o / rays_d / z_coarse is NULL");
  const bool perturb = (flags & DMNERF_FLAG_PERTURB) != 0;
  DMN_CHECK(!perturb || (io->t_rand && io->u), "render_forward: PERTURB needs t_rand and u");
  DMN_CHECK(io->z_row_stride == 0 || io->z_row_stride >= S, "render_forward: bad z_row_stride");
  cudaStream_t st = (cudaStream_t)stream;
  const int C = 4 + ctx->net[0].p.ins_num + 1, F = S + NI;
  const int keep_ins = (flags & DMNERF_FLAG_KEEP_INS) ? 1 : 0;
  DMN_CUDA(cudaSetDevice(ctx->device));
  if (resolve_impl(ctx, impl, 0, 1, st, "render_forward")) return 1;

  // ---- fully fused path: one launch, no intermediate tensor in HBM
  if (impl != DMNERF_IMPL_SIMT && S == 64 && NI == 128 && !io->raw_coarse && !io->raw_fine) {
    const bool prof = ctx->profiling;
    if (prof) DMN_CUDA(cudaEventRecord(ctx->ev[0], st));
    int rc = launch_render_tc(ctx->net[0], ctx->net[1], io, n, flags, st, edit, impl == DMNERF_IMPL_UMMA_F16);
    if (rc) return rc;
    if (prof) for (int i = 1; i <= DMNERF_N_STAGES; ++i) DMN_CUDA(cudaEventRecord(ctx->ev[i], st));
    ctx->profile_valid = prof;
    return 0;
  }

  // scratch for whatever the caller does not want back
  float* z_c = io->z_vals_coarse;
  if (!z_c && ctx->ws_z_c.get((size_t)n * S, &z_c)) return 2;
  float* z_f = io->z_vals_fine;
  if (!z_f && ctx->ws_z_f.get((size_t)n * F, &z_f)) return 2;
  float* w_c = io->weights_coarse;
  if (!w_c && ctx->ws_w_c.get((size_t)n * S, &w_c)) return 2;
  float* raw_c = io->raw_coarse;
  if (!raw_c && ctx->ws_raw_c.get((size_t)n * S * C, &raw_c)) return 2;
  float* raw_f = io->raw_fine;
  if (!raw_f && ctx->ws_raw_f.get((size_t)n * F * C, &raw_f)) return 2;

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
  if ((rc = launch_composite(raw_c, z_c, io->rays_d, n, S, C, keep_ins, io->rgb_coarse, w_c, io->depth_coarse,
                             io->ins_coarse, io->acc_coarse, st, edit, io->rays_o))) return rc;
  DMN_STAGE_MARK();
  // render.py:66-70  importance sampling + merge
  if ((rc = launch_hier_sample(z_c, w_c, perturb ? io->u : nullptr, n, S, NI, z_f, st))) return rc;
  DMN_STAGE_MARK();
  // render.py:71-82  fine network on all S+I depths
  if ((rc = mlp_dispatch(ctx, 1, nullptr, io->rays_o, io->rays_d, z_f, n * F, F, raw_f, impl, st))) return rc;
  DMN_STAGE_MARK();
  // render.py:86     fine composite
  if ((rc = launch_composite(raw_f, z_f, io->rays_d, n, F, C, keep_ins, io->rgb_fine, io->weights_fine, io->depth_fine,
                             io->ins_fine, io->acc_fine, st, edit, io->rays_o))) return rc;
  DMN_STAGE_MARK();
#undef DMN_STAGE_MARK
  ctx->profile_valid = prof;
  return 0;
}

extern "C" {

DMNERF_API int dmnerf_render_forward(dmnerf_ctx* ctx, const dmnerf_render_io* io, int64_t n, int S, int NI, int flags, int impl,
                          void* stream) {
  if (bound_pair(ctx, "render_forward")) return 1;
  DMN_CHECK(!(flags & ~RENDER_FLAGS), "render_forward: unknown flag bits 0x%x", flags & ~RENDER_FLAGS);
  Edit e;
  const Edit* edit;
  if (int rc = scene_edit(ctx, io ? io->edit : nullptr, (cudaStream_t)stream, e, edit, "render_forward")) return rc;
  return f16_verdict(ctx, render_forward_impl(ctx, io, n, S, NI, flags, impl, edit, stream), impl, stream);
}

DMNERF_API int dmnerf_sync_check(dmnerf_ctx* ctx, void* stream) {
  DMN_CHECK(ctx != nullptr, "sync_check: ctx is NULL");
  DMN_CUDA(cudaSetDevice(ctx->device));
  DMN_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  // fp16 range verdicts: taken from both weight sets (the stage path's coarse and fine networks each have an error word), so
  // that none is left behind for a later call, then reported after any protocol error
  const bool range0 = ctx->net[0].take_f16_range(), range1 = ctx->net[1].take_f16_range();
  for (const Network& n : ctx->net)
    if (int rc = n.check_status((cudaStream_t)stream)) return rc;
  DMN_CHECK(!range0 && !range1, "fp16 network: an activation exceeded the fp16 range (> 65504), so these results are invalid; "
            "render with the exact network (DMNERF_IMPL_UMMA)");
  return 0;
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

// Host-buffer render with the bound pair (bound_pair): `h` holds HOST pointers for the outputs (and for the inputs unless
// dev_rays_o / dev_rays_d are given: rays that are already resident on the device, e.g. generated there from the camera).
// edit: as for render_forward_impl, its appearance table already on the device, so that every part reads the one copy.
static int render_host_impl(dmnerf_ctx* ctx, const dmnerf_render_io* h, const float* dev_rays_o, const float* dev_rays_d, int64_t n,
                            int S, int NI, int flags, int impl, const Edit* edit, void* stream) {
  DMN_CHECK(h, "render_forward_host: io is NULL");
  DMN_CHECK(n >= 0, "render_forward_host: negative ray count");
  if (n == 0) return 0;
  const bool dev_rays = dev_rays_o != nullptr && dev_rays_d != nullptr;
  DMN_CHECK((dev_rays || (h->rays_o && h->rays_d)) && h->z_coarse, "render_forward_host: rays_o / rays_d / z_coarse is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  DMN_CUDA(cudaSetDevice(ctx->device));
  const int ins = ctx->net[0].p.ins_num, C = 4 + ins + 1, F = S + NI;
  const int n_ins_out = (flags & DMNERF_FLAG_KEEP_INS) ? ins + 1 : ins;
  const bool perturb = (flags & DMNERF_FLAG_PERTURB) != 0;
  const size_t zin = (h->z_row_stride == 0) ? (size_t)S : (size_t)n * h->z_row_stride;

  // ---- inputs: one device arena
  size_t in_floats = (dev_rays ? 0 : (size_t)n * 6) + zin + (perturb ? (size_t)n * (S + NI) : 0);
  float* d;
  if (ctx->host_in.get(in_floats, &d)) return 2;
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
  float* q;
  if (ctx->host_out.get(out_floats, &q)) return 2;
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
    int rc = render_forward_impl(ctx, &io, n, S, NI, flags, impl, edit, stream);
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
    rc = render_forward_impl(ctx, &pi, edge[i + 1] - edge[i], S, NI, flags, impl, edit, stream);
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
  if (bound_pair(ctx, "render_forward_host")) return 1;
  DMN_CHECK(!(flags & ~RENDER_FLAGS), "render_forward_host: unknown flag bits 0x%x", flags & ~RENDER_FLAGS);
  Edit e;
  const Edit* edit;
  if (int rc = scene_edit(ctx, h ? h->edit : nullptr, (cudaStream_t)stream, e, edit, "render_forward_host")) return rc;
  return render_host_impl(ctx, h, nullptr, nullptr, n, S, NI, flags, impl, edit, stream);
}

DMNERF_API int dmnerf_render_frame_host(dmnerf_ctx* ctx, const float* K_host, const float* c2w_host, int H, int W, float near_z,
                                        float far_z, int64_t ray_begin, int64_t ray_count, int n_coarse, int n_importance,
                                        int flags, int impl, const dmnerf_render_io* out_host, void* stream) {
  if (bound_pair(ctx, "render_frame_host")) return 1;
  DMN_CHECK(K_host && c2w_host && out_host, "render_frame_host: NULL argument");
  DMN_CHECK(!(flags & ~RENDER_FLAGS), "render_frame_host: unknown flag bits 0x%x", flags & ~RENDER_FLAGS);
  Edit e;
  const Edit* edit;
  if (int rc = scene_edit(ctx, out_host->edit, (cudaStream_t)stream, e, edit, "render_frame_host")) return rc;
  DMN_CHECK(H > 0 && W > 0 && n_coarse >= 3 && n_coarse <= 4096, "render_frame_host: bad sizes H=%d W=%d S=%d", H, W, n_coarse);
  DMN_CHECK(ray_begin >= 0 && ray_count >= 0 && ray_begin + ray_count <= (int64_t)H * W,
            "render_frame_host: pixel range [%lld, +%lld) outside the %dx%d frame", (long long)ray_begin, (long long)ray_count, H, W);
  DMN_CHECK(!(flags & DMNERF_FLAG_PERTURB), "render_frame_host: the frame driver is the deterministic test-time path");
  if (ray_count == 0) return 0;
  DMN_CUDA(cudaSetDevice(ctx->device));
  // rays of the whole frame on the device (helpers.py:50-61; tester.py:59-61), the range asked for is rendered
  float* ro;
  if (ctx->frame_rays.get((size_t)H * W * 6, &ro)) return 2;
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
  return render_host_impl(ctx, &h, ro + ray_begin * 3, rd + ray_begin * 3, ray_count, n_coarse, n_importance, flags, impl, edit,
                          stream);
}

// ---- mesh extraction (tools/mesh_generator.py mesh_main) ------------------------------------------------------------------

DMNERF_API int dmnerf_mesh_grid_points(const double* transform_host, const double* extents_host, int dim, int64_t begin, int64_t count,
                                       float* pts, void* stream) {
  DMN_CHECK(transform_host && extents_host && (count == 0 || pts), "mesh_grid_points: NULL argument");
  return launch_grid_points(transform_host, extents_host, dim, begin, count, pts, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_mesh_occupancy(dmnerf_ctx* ctx, int net, const double* transform_host, const double* extents_host, int dim,
                                     float voxel, int64_t slab, const uint32_t* keep_host, float* occ, int16_t* labels,
                                     void* stream) {
  if (bound_net(ctx, net, "mesh_occupancy")) return 1;
  DMN_CHECK(transform_host && extents_host && occ, "mesh_occupancy: NULL argument");
  DMN_CHECK(dim >= 2 && dim <= 2048, "mesh_occupancy: dim %d out of range [2, 2048]", dim);
  DMN_CHECK(keep_host || !labels, "mesh_occupancy: labels are written by the selected sweep only (pass keep_host)");
  ObjMask keep;
  if (object_mask(keep_host, ctx->net[net].p.ins_num + 1, keep, "mesh_occupancy")) return 1;
  cudaStream_t st = (cudaStream_t)stream;
  DMN_CUDA(cudaSetDevice(ctx->device));
  const int64_t n = (int64_t)dim * dim * dim;
  if (slab <= 0) slab = (int64_t)1 << 20;
  if (slab > n) slab = n;
  const int C = 4 + ctx->net[net].p.ins_num + 1;
  float *pts, *raw;
  if (ctx->mesh_pts.get((size_t)slab * 6, &pts) || ctx->mesh_raw.get((size_t)slab * C, &raw)) return 2;
  float* dirs = pts + slab * 3;                                   // mesh_generator.py:42: zero view directions
  DMN_CUDA(cudaMemsetAsync(dirs, 0, (size_t)slab * 3 * sizeof(float), st));
  // slab by slab: the [dim^3, C] network output of the original never exists, only [slab, C]
  for (int64_t b = 0; b < n; b += slab) {
    const int64_t cnt = n - b < slab ? n - b : slab;
    int rc = launch_grid_points(transform_host, extents_host, dim, b, cnt, pts, st);
    if (!rc) rc = launch_mlp_tc(ctx->net[net], nullptr, pts, dirs, nullptr, cnt, 1, raw, nullptr, st);
    if (!rc) rc = keep_host ? launch_occupancy_objects(raw, cnt, C, voxel, keep, occ + b, labels ? labels + b : nullptr, st)
                            : launch_occupancy(raw, cnt, C, voxel, occ + b, st);
    if (rc) return rc;
  }
  return 0;
}

DMNERF_API int dmnerf_mesh_occupancy_edit(dmnerf_ctx* ctx, int net, const double* transform_host, const double* extents_host, int dim,
                                          float voxel, float level, int64_t slab, const dmnerf_edit_move* moves_host, int n_moves,
                                          float* occ, int16_t* labels, int64_t* evaluated_host, void* stream) {
  const char* who = "mesh_occupancy_edit";
  if (bound_net(ctx, net, who)) return 1;
  if (evaluated_host) *evaluated_host = 0;
  DMN_CHECK(transform_host && extents_host && occ && labels, "%s: NULL argument", who);
  DMN_CHECK(dim >= 2 && dim <= 2048, "%s: dim %d out of range [2, 2048]", who, dim);
  DMN_CHECK(n_moves >= 0 && n_moves <= DMNERF_MAX_MOVES, "%s: between 0 and %d moves are supported, got %d", who, DMNERF_MAX_MOVES,
            n_moves);
  DMN_CHECK(n_moves == 0 || moves_host, "%s: moves is NULL", who);
  DMN_CHECK(level > 0.0f && level < 1.0f, "%s: level %g outside (0, 1)", who, (double)level);
  const double* T = transform_host;
  const double det = T[0] * (T[5] * T[10] - T[6] * T[9]) - T[1] * (T[4] * T[10] - T[6] * T[8]) + T[2] * (T[4] * T[9] - T[5] * T[8]);
  DMN_CHECK(det > 0.0, "%s: the scene transform has det %g <= 0", who, det);
  for (int a = 0; a < 3; ++a) DMN_CHECK(extents_host[a] > 0.0 && std::isfinite(extents_host[a]), "%s: extents must be finite and > 0", who);
  EditMove mv[DMNERF_MAX_MOVES];
  for (int i = 0; i < n_moves; ++i)
    if (edit_move_from_abi(moves_host[i], transform_host, extents_host, dim, ctx->net[net].p.ins_num, mv[i], who, i)) return 1;
  if (n_moves == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  DMN_CUDA(cudaSetDevice(ctx->device));
  const int64_t n = (int64_t)dim * dim * dim;
  if (slab <= 0) slab = (int64_t)1 << 20;
  if (slab > n) slab = n;
  const int C = 4 + ctx->net[net].p.ins_num + 1;
  float *pts, *raw;
  if (ctx->mesh_pts.get((size_t)slab * 6, &pts) || ctx->mesh_raw.get((size_t)slab * C, &raw)) return 2;
  float* dirs = pts + slab * 3;                                   // zero view directions, as the sweep
  DMN_CUDA(cudaMemsetAsync(dirs, 0, (size_t)slab * 3 * sizeof(float), st));
  int64_t evaluated = 0;
  // slab by slab, move by move: a point's moves only read its own earlier state, so this is the moves applied in order
  for (int64_t b = 0; b < n; b += slab) {
    const int64_t cnt = n - b < slab ? n - b : slab;
    for (int i = 0; i < n_moves; ++i) {
      int64_t m = 0;
      int rc = edit_targets(ctx->mesh, transform_host, extents_host, dim, mv[i], b, cnt, pts, &m, st);
      if (!rc && m) rc = launch_mlp_tc(ctx->net[net], nullptr, pts, dirs, nullptr, m, 1, raw, nullptr, st);
      if (!rc) rc = edit_apply(ctx->mesh, transform_host, extents_host, dim, mv[i], b, cnt, raw, C, voxel, level, occ, labels, st);
      if (rc) return rc;
      evaluated += m;
    }
  }
  if (evaluated_host) *evaluated_host = evaluated;
  return 0;
}

DMNERF_API int dmnerf_mesh_vertex_labels(const float* verts, int64_t n, const float* occ, const int16_t* labels, int dim, float level,
                                         int16_t* out, void* stream) {
  return launch_vertex_labels(verts, n, occ, labels, dim, level, out, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_mesh_mc_count(dmnerf_ctx* ctx, const float* grid, int nx, int ny, int nz, float level, int64_t* counts_host,
                                    void* stream) {
  DMN_CHECK(ctx && grid && counts_host, "mesh_mc_count: NULL argument");
  DMN_CUDA(cudaSetDevice(ctx->device));
  return mc_count(ctx->mesh, grid, nx, ny, nz, level, counts_host, (cudaStream_t)stream);
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
  return mesh_normals(ctx->mesh, verts, nv, tris, nt, normals, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_mesh_clusters(dmnerf_ctx* ctx, const int32_t* tris, int64_t nt, int64_t nv, int32_t* cluster, int32_t* cluster_size,
                                    void* stream) {
  DMN_CHECK(ctx && (nt == 0 || (tris && cluster && cluster_size)), "mesh_clusters: NULL argument");
  DMN_CUDA(cudaSetDevice(ctx->device));
  return mesh_clusters(ctx->mesh, tris, nt, nv, cluster, cluster_size, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_mesh_clean(dmnerf_ctx* ctx, const float* verts, const float* normals, int64_t nv, const int32_t* tris, int64_t nt,
                                 const int32_t* cluster_size, int min_cluster, float* out_verts, float* out_normals, int32_t* out_tris,
                                 int64_t* counts_host, void* stream) {
  DMN_CHECK(ctx && counts_host, "mesh_clean: NULL argument");
  DMN_CHECK(nv == 0 || (verts && out_verts && (!normals == !out_normals)), "mesh_clean: NULL vertex buffer");
  DMN_CHECK(nt == 0 || (tris && cluster_size && out_tris), "mesh_clean: NULL triangle buffer");
  DMN_CUDA(cudaSetDevice(ctx->device));
  return mesh_clean(ctx->mesh, verts, normals, nv, tris, nt, cluster_size, min_cluster, out_verts, out_normals, out_tris, counts_host,
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

// ---- object inventory (DESIGN.md, "Object inventory") ---------------------------------------------------------------------

DMNERF_API int dmnerf_object_voxels(dmnerf_ctx* ctx, const float* occ, const int16_t* labels, int dim, float level, int n_labels,
                                    const int32_t* boxes_host, int64_t* moments_host, uint32_t* hist_host, void* stream) {
  DMN_CHECK(ctx != nullptr, "object_voxels: ctx is NULL");
  DMN_CUDA(cudaSetDevice(ctx->device));
  return object_voxels(ctx->inventory, occ, labels, dim, level, n_labels, boxes_host, moments_host, hist_host, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_object_spans(dmnerf_ctx* ctx, const float* occ, const int16_t* labels, int dim, float level, int n_labels,
                                   const int32_t* boxes_host, const double* axes_host, double* spans_host, void* stream) {
  DMN_CHECK(ctx != nullptr, "object_spans: ctx is NULL");
  DMN_CUDA(cudaSetDevice(ctx->device));
  return object_spans(ctx->inventory, occ, labels, dim, level, n_labels, boxes_host, axes_host, spans_host, (cudaStream_t)stream);
}

// ---- connected components (DESIGN.md, "Connected components") -------------------------------------------------------------

DMNERF_API int dmnerf_object_components(dmnerf_ctx* ctx, const float* occ, const int16_t* labels, int dim, float level, int n_labels,
                                        int connectivity, int32_t* comp, int64_t* n_components_host, void* stream) {
  DMN_CHECK(ctx != nullptr, "object_components: ctx is NULL");
  DMN_CUDA(cudaSetDevice(ctx->device));
  return object_components(ctx->components, occ, labels, dim, level, n_labels, connectivity, comp, n_components_host,
                           (cudaStream_t)stream);
}

DMNERF_API int dmnerf_component_table(dmnerf_ctx* ctx, const int32_t* comp, const int16_t* labels, int dim, int64_t n, int16_t* label,
                                      int64_t* voxels, int64_t* root, void* stream) {
  DMN_CHECK(ctx != nullptr, "component_table: ctx is NULL");
  DMN_CUDA(cudaSetDevice(ctx->device));
  return component_table(ctx->components, comp, labels, dim, n, label, voxels, root, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_component_groups(dmnerf_ctx* ctx, const int32_t* comp, int dim, int64_t n, const int16_t* lut, int discard,
                                       int16_t* groups, void* stream) {
  DMN_CHECK(ctx != nullptr, "component_groups: ctx is NULL");
  DMN_CUDA(cudaSetDevice(ctx->device));
  return component_groups(ctx->components, comp, dim, n, lut, discard, groups, (cudaStream_t)stream);
}

// ---- region selection (DESIGN.md, "Region selection") ---------------------------------------------------------------------

DMNERF_API int dmnerf_region_pack(const int32_t* ids, int dim, const uint32_t* table, int64_t n_ids, uint32_t* bits, void* stream) {
  return region_pack(ids, dim, table, n_ids, bits, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_region_dilate(dmnerf_ctx* ctx, const uint32_t* in, int dim, int radius, int connectivity, int invert,
                                    uint32_t* out, void* stream) {
  DMN_CHECK(ctx != nullptr, "region_dilate: ctx is NULL");
  DMN_CUDA(cudaSetDevice(ctx->device));
  if (region_check(dim, nullptr, "region_dilate")) return 1;
  uint32_t* tmp = nullptr;
  if (radius >= 2 && ctx->region_tmp.get((size_t)region_words(dim), &tmp)) return 2;
  return region_dilate(in, dim, radius, connectivity, invert, out, tmp, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_region_contains(const dmnerf_region* region, const float* pts, int64_t n, uint8_t* out, void* stream) {
  DMN_CHECK(region != nullptr, "region_contains: region is NULL");
  Region r;
  if (region_from_abi(*region, r, "region_contains")) return 1;
  return region_contains(r, pts, n, out, (cudaStream_t)stream);
}

// ---- test-view evaluation (networks/tester.py render_test, networks/evaluator.py ins_eval) --------------------------------

DMNERF_API int64_t dmnerf_eval_workspace_bytes(int64_t n, int k, int H, int W) {
  if (n < 0 || k < 0 || H < 0 || W < 0) return -1;
  return eval_workspace_bytes(n, k, H, W);
}

DMNERF_API int dmnerf_eval_image(const float* rgb, const float* gt, int H, int W, void* ws, dmnerf_eval_result* res, void* stream) {
  DMN_CHECK(rgb && gt && ws && res, "eval_image: NULL argument");
  return eval_image(rgb, gt, H, W, ws, res, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_ins_eval(const float* ins, int64_t n, int k, const int32_t* gt_row, int gt_num, const float* mask,
                               const int32_t* mask_labels, int mask_below, int64_t* pred_label, void* ws, dmnerf_eval_result* res,
                               void* stream) {
  DMN_CHECK(ins && gt_row && pred_label && ws && res, "ins_eval: NULL argument");
  DMN_CHECK(!(mask && mask_labels), "ins_eval: pass either mask or mask_labels, not both");
  return ins_eval(ins, n, k, gt_row, gt_num, mask, mask_labels, mask_below, pred_label, ws, res, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_calculate_ap(const float* ious, const float* conf, int m, int gt_number, float* ap6, void* stream) {
  DMN_CHECK(ious && ap6, "calculate_ap: NULL argument");
  return calculate_ap(ious, conf, m, gt_number, ap6, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_ins_dense_rows(const float* gt_ins, int64_t n, int k, int gt_num, int32_t* gt_row, void* stream) {
  DMN_CHECK(n >= 0 && k >= 1 && (n == 0 || (gt_ins && gt_row)), "ins_dense_rows: bad argument");
  return ins_dense_rows(gt_ins, n, k, gt_num, gt_row, (cudaStream_t)stream);
}

DMNERF_API int dmnerf_label_colors(const void* labels, int labels_are_64bit, int64_t n, const uint8_t* lut, int n_lut, uint8_t* out,
                                   void* stream) {
  DMN_CHECK(n >= 0 && n_lut >= 0 && (n == 0 || (labels && out)) && (n_lut == 0 || lut), "label_colors: bad argument");
  return label_colors(labels, labels_are_64bit, n, lut, n_lut, out, (cudaStream_t)stream);
}

}  // extern "C"
