"""Object manipulation at render time (reference networks/manipulator.py:18-205) on the native kernels: the four functions
of the edit path with the reference's names and signatures.

    exchanger(ori_raw, tar_raws, ori_raw_pred, tar_raw_preds, move_labels)               manipulator.py:18-83   (one kernel)
    manipulator_render(raw, z_vals, rays_d)                                              manipulator.py:86-105  (composite, all instance channels)
    manipulator_nerf(rays, position_embedder, view_embedder, model, N_samples, near, far, z_vals)   manipulator.py:108-134 (tensor-core network)
    manipulator(position_embedder, view_embedder, model_coarse, model_fine, ori_rays, f_tar_rays, args)   manipulator.py:137-205

The evaluation / demo loops of the reference module (image IO, metrics) are not part of the path and are not provided.
"""
import ctypes as C

import torch

from . import _lib
from .engine import get_context
from .autograd import mlp_forward_rays
from .render import composite, _check_embedders
from .helpers import sample_pdf, sort_concat


def exchanger(ori_raw, tar_raws, ori_raw_pred, tar_raw_preds, move_labels):
    """Edits `ori_raw` in place like the reference and returns (ori_raw, tar_raws, ori_pred_label, tar_pred_label)."""
    if not ori_raw.is_cuda:
        raise RuntimeError("exchanger: expected CUDA tensors (no CPU fallback)")
    if not (ori_raw.is_contiguous() and ori_raw.dtype == torch.float32):
        raise RuntimeError("exchanger: ori_raw must be a contiguous float32 tensor (it is edited in place)")
    n, s, c = ori_raw.shape
    m = len(move_labels)
    tars = [t.contiguous().float() for t in tar_raws]
    accs = [a.contiguous().float() for a in tar_raw_preds]
    acc_o = ori_raw_pred.contiguous().float()
    if len(tars) < m or len(accs) < m or any(t.shape != ori_raw.shape for t in tars[:m]) or acc_o.shape != (n, c - 4):
        raise RuntimeError("exchanger: inconsistent shapes")
    ctx = get_context(ori_raw.device)
    ori_label = torch.empty((n, s), device=ori_raw.device, dtype=torch.int64)
    tar_label = torch.empty((n, s), device=ori_raw.device, dtype=torch.int64)
    tp = (C.c_void_p * m)(*[t.data_ptr() for t in tars[:m]])
    ap = (C.c_void_p * m)(*[a.data_ptr() for a in accs[:m]])
    mv = (C.c_int * m)(*[int(v) for v in move_labels])
    _lib.check(ctx.lib.dmnerf_exchanger(_lib.ptr(ori_raw), tp, _lib.ptr(acc_o), ap, mv, m, n, s, c, ori_label.data_ptr(),
                                        tar_label.data_ptr(), ctx.stream()), "dmnerf_exchanger")
    return ori_raw, tar_raws, ori_label, tar_label


def manipulator_render(raw, z_vals, rays_d):
    rgb, weights, depth, ins, _ = composite(raw, z_vals, rays_d, keep_all_ins=True)
    return rgb, weights, depth, ins


def manipulator_nerf(rays, position_embedder, view_embedder, model, N_samples=None, near=None, far=None, z_vals=None,
                     impl=_lib.IMPL_AUTO):
    _check_embedders(position_embedder, view_embedder)
    rays_o, rays_d = rays
    n = rays_d.shape[0]
    if z_vals is None:
        dev = rays_d.device
        near_, far_ = near * torch.ones(size=(n, 1), device=dev), far * torch.ones(size=(n, 1), device=dev)
        t_vals = torch.linspace(0., 1., steps=N_samples, device=dev)
        z_vals = (near_ * (1. - t_vals) + far_ * t_vals).expand([n, N_samples])       # manipulator.py:117-120
    raw = mlp_forward_rays(model, rays_o, rays_d, z_vals.contiguous(), impl)
    return raw, z_vals


def manipulator(position_embedder, view_embedder, model_coarse, model_fine, ori_rays, f_tar_rays, args, us=None,
                impl=_lib.IMPL_AUTO):
    """manipulator.py:137-205.  `us`: optional list of [N, N_importance] uniforms replacing the torch.rand draws of the
    sample_pdf calls (order: original rays, every target, original rays again) -- used by the parity tests."""
    N_samples, N_importance, near, far = args.N_samples, args.N_importance, args.near, args.far
    us = list(us) if us is not None else None

    def draw(bins, w):
        return sample_pdf(bins, w, N_importance, u=(us.pop(0) if us is not None else None))

    def nerf(rays, model, z=None):
        return manipulator_nerf(rays, position_embedder, view_embedder, model, N_samples, near, far, z_vals=z, impl=impl)

    def fine_pass(rays, coarse_raw, coarse_z):
        _, w, _, _ = manipulator_render(coarse_raw, coarse_z, rays[1])
        mid = .5 * (coarse_z[..., 1:] + coarse_z[..., :-1])
        z_s = draw(mid, w[..., 1:-1])
        z_full = sort_concat(coarse_z, z_s)                                   # sort(cat(.)) as one kernel
        raw_full, _ = nerf(rays, model_fine, z_full)
        _, _, _, ins_acc = manipulator_render(raw_full, z_full, rays[1])
        return z_s, ins_acc

    with torch.no_grad():
        ori_raw, ori_z = nerf(ori_rays, model_coarse)
        _, ori_ins_acc = fine_pass(ori_rays, ori_raw, ori_z)
        tar_raws, tar_zs, tar_samples, tar_accs = [], [], [], []
        tar_rgb = None
        for tar_rays in f_tar_rays:
            t_raw, t_z = nerf(tar_rays, model_coarse)
            tar_rgb, _, _, _ = manipulator_render(t_raw, t_z, tar_rays[1])
            z_s, acc = fine_pass(tar_rays, t_raw, t_z)
            tar_raws.append(t_raw); tar_zs.append(t_z); tar_samples.append(z_s); tar_accs.append(acc)
        ori_raw, _, _, _ = exchanger(ori_raw, tar_raws, ori_ins_acc, tar_accs, args.target_labels)
        _, ori_w, _, _ = manipulator_render(ori_raw, ori_z, ori_rays[1])
        mid = .5 * (ori_z[..., 1:] + ori_z[..., :-1])
        ori_samples = draw(mid, ori_w[..., 1:-1])
        extra = torch.cat([ori_samples] + tar_samples, -1)                     # samples every second-pass ray set shares
        ori_z2 = sort_concat(ori_z, extra)
        ori_raw2, _ = nerf(ori_rays, model_fine, ori_z2)
        for idx, tar_rays in enumerate(f_tar_rays):
            t_z2 = sort_concat(tar_zs[idx], extra)
            tar_raws[idx], _ = nerf(tar_rays, model_fine, t_z2)
        ori_raw2, _, _, _ = exchanger(ori_raw2, tar_raws, ori_ins_acc, tar_accs, args.target_labels)
        final_rgb, _, _, final_ins = manipulator_render(ori_raw2, ori_z2, ori_rays[1])
    return final_rgb, final_ins, tar_rgb, tar_accs[-1]
