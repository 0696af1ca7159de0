"""Differentiable entry points (torch.autograd.Function over the native forward/backward kernels).

The training forward evaluates the networks with the tensor-core kernel (or the exact-fp32 CUDA-core kernel, see
TRAIN_IMPL) and keeps the activations the backward needs (dmnerf_mlp_forward_train); the backward is composite_backward
(closed-form reverse scan) followed by dmnerf_mlp_backward (heads folded like in the forward, one masked wgmma GEMM per
trunk layer, batched wgmma weight gradients).  Gradient topology is the reference's (SURVEY.md 3.3): no gradient through sample_pdf
(render.py:68), the instance map sees detached weights (render.py:22-23), the instance branch sees h.detach()
(dm_nerf.py:95), rays / depths carry no gradient.
"""
import os

import torch

from . import _lib
from .engine import get_context, ordered_params
from .render import bind_pair, coarse_depths, reference_draws

# Kernel used by the training forward: the tensor-core kernel by default ("umma"), or the exact-fp32 CUDA-core kernel ("simt").
TRAIN_IMPL = _lib.IMPL_SIMT if os.environ.get("DMNERF_TRAIN_IMPL", "umma").lower() == "simt" else _lib.IMPL_UMMA


def _train_impl(impl):
    if impl == _lib.IMPL_UMMA_F16:
        raise RuntimeError("IMPL_UMMA_F16 is inference-only: training and its gradients run the exact network (IMPL_UMMA or "
                           "IMPL_SIMT); call under torch.no_grad() for an fp16 preview")
    return TRAIN_IMPL if impl == _lib.IMPL_AUTO else impl


def _f32(t):
    return t.contiguous().float()


def _zeros_like_params(params):
    """One zero-filled flat buffer with a view per parameter (one fill kernel instead of 30 memsets); views start 16-byte
    aligned."""
    offs, total = [], 0
    for p in params:
        offs.append(total)
        total += (p.numel() + 3) // 4 * 4
    flat = torch.zeros(total, device=params[0].device, dtype=torch.float32)
    return [flat[o:o + p.numel()].view(p.shape) for o, p in zip(offs, params)]


def _mlp_backward(ctx, slot, acts, d_out, m, params, masks_saved):
    grads = _zeros_like_params(params)
    flags = int(masks_saved) | 2            # bit 0 = ReLU bit planes saved by the forward, bit 1 = gradient buffers already zero
    n_scratch = int(ctx.lib.dmnerf_mlp_backward_scratch_floats(m))
    scratch = torch.empty(max(n_scratch, 1), device=d_out.device, dtype=torch.float32)
    ctx.call("dmnerf_mlp_backward", ctx.handle, slot, _lib.ptr(acts), _lib.ptr(d_out), m, _lib.ptrs(grads), _lib.ptr(scratch),
             flags)
    return grads


class MLPFunction(torch.autograd.Function):
    """DM_NeRF.forward (networks/dm_nerf.py:80-106) with gradients w.r.t. the 30 parameters (not w.r.t. x: the reference
    never differentiates through the embedded inputs)."""

    @staticmethod
    def forward(fctx, model, x, impl, *params):
        ctx = get_context(x.device)
        slot = ctx.slot_for(model)
        ins_num = ctx.bind(slot, model)
        x2 = _f32(x.reshape(-1, x.shape[-1]))
        m = x2.shape[0]
        out = torch.empty((m, 4 + ins_num + 1), device=x.device, dtype=torch.float32)
        acts = torch.empty(max(m * ctx.lib.dmnerf_act_floats_per_sample(), 1), device=x.device, dtype=torch.float32)
        impl = _train_impl(impl)
        ctx.call("dmnerf_mlp_forward_train", ctx.handle, slot, _lib.ptr(x2), None, None, None, m, 1, _lib.ptr(out), _lib.ptr(acts),
                 impl)
        fctx.model, fctx.m, fctx.acts, fctx.params, fctx.masks_saved = model, m, acts, params, impl != _lib.IMPL_SIMT
        return out.reshape(*x.shape[:-1], out.shape[-1])

    @staticmethod
    def backward(fctx, g_out):
        ctx = get_context(g_out.device)
        slot = ctx.slot_for(fctx.model)
        ctx.bind(slot, fctx.model)
        d_out = _f32(g_out.reshape(fctx.m, -1))
        grads = _mlp_backward(ctx, slot, fctx.acts, d_out, fctx.m, fctx.params, fctx.masks_saved)
        return (None, None, None) + tuple(grads)


def mlp_forward_grad(model, x, impl=_lib.IMPL_AUTO):
    params, _ = ordered_params(model)
    return MLPFunction.apply(model, x, impl, *params)


class CompositeFunction(torch.autograd.Function):
    """render_train (networks/render.py:6-28) with gradient w.r.t. raw."""

    @staticmethod
    def forward(fctx, raw, z_vals, rays_d, keep_all_ins):
        from .render import composite
        raw, z_vals, rays_d = _f32(raw), _f32(z_vals), _f32(rays_d)
        rgb, w, depth, ins, _acc = composite(raw, z_vals, rays_d, keep_all_ins)
        fctx.save_for_backward(raw, z_vals, rays_d)
        fctx.keep = bool(keep_all_ins)
        return rgb, w, depth, ins

    @staticmethod
    def backward(fctx, g_rgb, g_w, g_depth, g_ins):
        raw, z, rd = fctx.saved_tensors
        n, s, c = raw.shape
        ctx = get_context(raw.device)
        d_raw = torch.empty_like(raw)
        # converted grads stay alive across the launch (a stride-0 expand from .sum().backward() is copied by _f32)
        keep = [_f32(g) if g is not None else None for g in (g_rgb, g_depth, g_ins, g_w)]
        ctx.call("dmnerf_composite_backward", _lib.ptr(raw), _lib.ptr(z), _lib.ptr(rd), n, s, c, int(fctx.keep), _lib.ptr(keep[0]),
                 _lib.ptr(keep[1]), None, _lib.ptr(keep[2]), _lib.ptr(keep[3]), _lib.ptr(d_raw), 0)
        return d_raw, None, None, None


_OUT_KEYS = ("rgb_coarse", "rgb_fine", "ins_coarse", "ins_fine", "depth_coarse", "depth_fine", "acc_coarse", "acc_fine",
             "raw_coarse", "raw_fine", "weights_coarse", "weights_fine", "z_vals_coarse", "z_vals_fine")


class RenderFunction(torch.autograd.Function):
    """dm_nerf() (networks/render.py:31-96) for training: forward + backward through both networks."""

    @staticmethod
    def forward(fctx, model_c, model_f, rays_o, rays_d, z_in, z_stride, t_rand, u, n_importance, n_c, impl, *params):
        dev = rays_o.device
        ctx = get_context(dev)
        impl = _train_impl(impl)
        ins_num = bind_pair(ctx, model_c, model_f)
        n, S = rays_o.shape[0], z_in.shape[-1]
        F, Cc = S + n_importance, 4 + ins_num + 1
        e = lambda *shape: torch.empty(shape, device=dev, dtype=torch.float32)
        apf = ctx.lib.dmnerf_act_floats_per_sample()
        o = {}
        # render.py:40-47 coarse depths
        o["z_vals_coarse"] = e(n, S)
        ctx.call("dmnerf_stratify", _lib.ptr(z_in), z_stride, _lib.ptr(t_rand), n, S, _lib.ptr(o["z_vals_coarse"]))
        saved = []
        for net, zkey, tag, ns in ((0, "z_vals_coarse", "coarse", S), (1, "z_vals_fine", "fine", F)):
            if net == 1:       # render.py:66-70 importance sampling on the (detached) coarse weights
                o["z_vals_fine"] = e(n, F)
                ctx.call("dmnerf_hier_sample", _lib.ptr(o["z_vals_coarse"]), _lib.ptr(o["weights_coarse"]), _lib.ptr(u), n, S,
                         n_importance, _lib.ptr(o["z_vals_fine"]))
            raw = e(n, ns, Cc)
            acts = e(max(n * ns * apf, 1))
            ctx.call("dmnerf_mlp_forward_train", ctx.handle, net, None, _lib.ptr(rays_o), _lib.ptr(rays_d), _lib.ptr(o[zkey]), n * ns,
                     ns, _lib.ptr(raw), _lib.ptr(acts), impl)
            rgb, w, depth, acc, ins = e(n, 3), e(n, ns), e(n), e(n), e(n, ins_num)
            ctx.call("dmnerf_composite", _lib.ptr(raw), _lib.ptr(o[zkey]), _lib.ptr(rays_d), n, ns, Cc, 0, None, _lib.ptr(rgb),
                     _lib.ptr(w), _lib.ptr(depth), _lib.ptr(ins), _lib.ptr(acc))
            o["raw_" + tag], o["rgb_" + tag], o["weights_" + tag] = raw, rgb, w
            o["depth_" + tag], o["acc_" + tag], o["ins_" + tag] = depth, acc, ins
            saved.append(acts)
        fctx.models = (model_c, model_f)
        fctx.n, fctx.S, fctx.F, fctx.C, fctx.n_c = n, S, F, Cc, n_c
        fctx.acts = saved
        fctx.masks_saved = impl != _lib.IMPL_SIMT
        fctx.params = params
        fctx.save_for_backward(rays_d, o["z_vals_coarse"], o["z_vals_fine"], o["raw_coarse"], o["raw_fine"])
        outs = tuple(o[k] for k in _OUT_KEYS)
        fctx.mark_non_differentiable(o["z_vals_coarse"], o["z_vals_fine"])
        return outs

    @staticmethod
    def backward(fctx, *g):
        gd = dict(zip(_OUT_KEYS, g))
        rays_d, z_c, z_f, raw_c, raw_f = fctx.saved_tensors
        ctx = get_context(rays_d.device)
        ctx.bind(0, fctx.models[0]); ctx.bind(1, fctx.models[1])
        n, Cc = fctx.n, fctx.C
        all_grads = []
        for net, tag, z, raw, ns in ((0, "coarse", z_c, raw_c, fctx.S), (1, "fine", z_f, raw_f, fctx.F)):
            g_raw = gd["raw_" + tag]
            if g_raw is not None:
                d_raw, accumulate = _f32(g_raw).clone(), 1
            else:
                d_raw, accumulate = torch.empty_like(raw), 0
            keep = [_f32(gd[k + tag]) if gd[k + tag] is not None else None for k in ("rgb_", "depth_", "acc_", "ins_", "weights_")]
            ctx.call("dmnerf_composite_backward", _lib.ptr(raw), _lib.ptr(z), _lib.ptr(rays_d), n, ns, Cc, 0, _lib.ptr(keep[0]),
                     _lib.ptr(keep[1]), _lib.ptr(keep[2]), _lib.ptr(keep[3]), _lib.ptr(keep[4]), _lib.ptr(d_raw), accumulate)
            params = fctx.params[:fctx.n_c] if net == 0 else fctx.params[fctx.n_c:]
            all_grads += _mlp_backward(ctx, net, fctx.acts[net], d_raw.reshape(n * ns, Cc), n * ns, params, fctx.masks_saved)
        fctx.acts = None
        return (None,) * 11 + tuple(all_grads)


def render_rays_grad(rays_o, rays_d, model_coarse, model_fine, z_vals_coarse, perturb=0.0, N_importance=128,
                     t_rand=None, u=None, impl=_lib.IMPL_AUTO):
    """Training-mode dm_nerf(): same dict as render.render_rays, differentiable w.r.t. both networks' parameters."""
    dev = rays_o.device
    if dev.type != "cuda":
        raise RuntimeError("dm_nerf: expected CUDA tensors (no CPU fallback)")
    rays_o, rays_d = _f32(rays_o.reshape(-1, 3)), _f32(rays_d.reshape(-1, 3))
    n = rays_o.shape[0]
    z_in, z_stride = coarse_depths(z_vals_coarse, n)
    t_rand, u = reference_draws(perturb, n, z_vals_coarse.shape[-1], N_importance, dev, t_rand, u)
    pc, _ = ordered_params(model_coarse)
    pf, _ = ordered_params(model_fine)
    outs = RenderFunction.apply(model_coarse, model_fine, rays_o, rays_d, z_in, z_stride, t_rand, u, N_importance, len(pc),
                                _train_impl(impl), *pc, *pf)
    return dict(zip(_OUT_KEYS, outs))
