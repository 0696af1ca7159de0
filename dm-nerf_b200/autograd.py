"""torch entry points of the native kernels.  Inference (torch.no_grad / no parameter requires grad)
goes straight to the C ABI; the differentiable variants are torch.autograd.Function wrappers."""
import torch

from . import _lib
from .engine import get_context


def _needs_grad(*models_and_tensors):
    if not torch.is_grad_enabled():
        return False
    for m in models_and_tensors:
        if isinstance(m, torch.nn.Module):
            if any(p.requires_grad for p in m.parameters()):
                return True
        elif torch.is_tensor(m) and m.requires_grad:
            return True
    return False


def mlp_forward(model, x, impl=_lib.IMPL_AUTO):
    """DM_NeRF.forward (networks/dm_nerf.py:80-106): x [..., 90] -> [..., 4 + ins_num + 1]."""
    if not x.is_cuda:
        raise RuntimeError("DM_NeRF.forward: expected a CUDA tensor (no CPU fallback)")
    if _needs_grad(model, x):
        from .backward import mlp_forward_grad
        return mlp_forward_grad(model, x, impl)
    impl = _lib.infer_impl(impl)
    ctx = get_context(x.device)
    slot = ctx.slot_for(model)
    ins_num = ctx.bind(slot, model)
    x2 = x.reshape(-1, x.shape[-1]).contiguous().float()
    if x2.shape[1] != 90:
        raise RuntimeError("DM_NeRF.forward: expected 90 input channels (63 pos + 27 dir), got %d" % x2.shape[1])
    out = torch.empty((x2.shape[0], 4 + ins_num + 1), device=x.device, dtype=torch.float32)
    ctx.call("dmnerf_mlp_forward", ctx.handle, slot, _lib.ptr(x2), x2.shape[0], _lib.ptr(out), impl)
    return out.reshape(*x.shape[:-1], out.shape[-1])


def mlp_forward_rays(model, rays_o, rays_d, z, impl=_lib.IMPL_AUTO):
    """Network evaluated at pts = o + d*z with both embeddings fused in (render.py:49-61).  Inference only."""
    impl = _lib.infer_impl(impl)
    ctx = get_context(z.device)
    slot = ctx.slot_for(model)
    ins_num = ctx.bind(slot, model)
    n, s = z.shape
    # the converted copies must outlive the launch: a temporary freed inside the argument list would hand its block to the next
    # same-size temporary in the caching allocator (rays_o aliasing rays_d)
    ro, rd, zz = rays_o.reshape(-1, 3).contiguous().float(), rays_d.reshape(-1, 3).contiguous().float(), z.contiguous().float()
    if ro.shape[0] != n or rd.shape[0] != n:
        raise RuntimeError("mlp_forward_rays: %d / %d rays for %d depth rows" % (ro.shape[0], rd.shape[0], n))
    out = torch.empty((n, s, 4 + ins_num + 1), device=z.device, dtype=torch.float32)
    ctx.call("dmnerf_mlp_forward_rays", ctx.handle, slot, _lib.ptr(ro), _lib.ptr(rd), _lib.ptr(zz), n, s, _lib.ptr(out), impl)
    return out


def mlp_forward_points(model, pts, viewdirs=None, impl=_lib.IMPL_AUTO):
    """The network at arbitrary points with explicit view directions (zeros by default), embedded inside the kernel: the grid
    sweep of tools/mesh_generator.py:36-49.  pts [..., 3] -> [..., 4 + ins_num + 1]."""
    if not pts.is_cuda:
        raise RuntimeError("mlp_forward_points: expected CUDA tensors (no CPU fallback)")
    impl = _lib.infer_impl(impl)
    ctx = get_context(pts.device)
    slot = ctx.slot_for(model)
    ins_num = ctx.bind(slot, model)
    p2 = pts.reshape(-1, 3).contiguous().float()
    v2 = torch.zeros_like(p2) if viewdirs is None else viewdirs.reshape(-1, 3).contiguous().float()
    out = torch.empty((p2.shape[0], 4 + ins_num + 1), device=pts.device, dtype=torch.float32)
    ctx.call("dmnerf_mlp_forward_points", ctx.handle, slot, _lib.ptr(p2), _lib.ptr(v2), p2.shape[0], _lib.ptr(out), impl)
    return out.reshape(*pts.shape[:-1], out.shape[-1])
