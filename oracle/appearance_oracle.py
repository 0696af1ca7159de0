"""CPU oracle of object appearance -- TEST INFRASTRUCTURE ONLY (the product package never imports it).

Restates DESIGN.md, "Object appearance" in torch, one rounding per operation (CPU elementwise ops neither contract nor widen).
An appearance is a table [ins_num + 1, 16] (objects.Appearance.table): per label l the colour map [M_l | b_l] (row-major 3x4),
the density scale s_l and 3 floats of padding.  Per sample with label l (objects_oracle.object_labels), after the label
selection and the region's exclusion:
  density  raw[..., 3] becomes s_l relu(raw[..., 3]), one product: the composite's relu leaves it as it is, and an excluded
           sample (density 0) stays at alpha = 0;
  colour   c = sigmoid(raw[..., :3]); c'_a = clamp(((M_a0 c0 + M_a1 c1) + M_a2 c2) + b_a, 0, 1); rgb = sum_i w_i c'_i.
Depth, acc and the instance maps are the composite's own, on the edited weights.  `render` and `render_on_depths` are
region_oracle's, with the appearance as one more optional argument; without one they return what those do."""
import numpy as np
import torch


def _table(appearance, like):
    t = getattr(appearance, "table", appearance)
    return torch.as_tensor(np.asarray(t, dtype=np.float32)).to(dtype=like.dtype, device=like.device)


def scale_density(raw, labels, appearance):
    """raw with raw[..., 3] = s_label relu(raw[..., 3]) (a new tensor)."""
    s = _table(appearance, raw)[:, 12]
    out = raw.clone()
    out[..., 3] = s[labels.to(raw.device)] * torch.relu(raw[..., 3])
    return out


def edited_colour(raw, labels, appearance):
    """The per-sample colour c' [..., 3] of the rule from the network's raw rgb."""
    m = _table(appearance, raw)[:, :12].reshape(-1, 3, 4)[labels.to(raw.device)]          # [..., 3, 4]
    c = torch.sigmoid(raw[..., :3])
    u = [((m[..., a, 0] * c[..., 0] + m[..., a, 1] * c[..., 1]) + m[..., a, 2] * c[..., 2]) + m[..., a, 3] for a in range(3)]
    return torch.clamp(torch.stack(u, -1), 0.0, 1.0)


def composite(raw, raw_sel, z, rays_d, appearance=None, keep_all_ins=False):
    """dmnerf_oracle.composite of raw_sel (raw after the selection and the exclusion) with the appearance: the density scaled
    before, the rgb map taken over the edited colours of raw.  (rgb, weights, depth, ins, acc)."""
    from . import dmnerf_oracle as O
    from . import objects_oracle as OO
    if appearance is None:
        return O.composite(raw_sel, z, rays_d, keep_all_ins=keep_all_ins)
    labels = OO.object_labels(raw)
    rgb, w, depth, ins, acc = O.composite(scale_density(raw_sel, labels, appearance), z, rays_d, keep_all_ins=keep_all_ins)
    rgb = torch.sum(w[..., None] * edited_colour(raw, labels, appearance), -2)
    return rgb, w, depth, ins, acc


def render(rays_o, rays_d, p_coarse, p_fine, z_coarse, keep, perturb=0.0, n_importance=128, t_rand=None, u=None, exclude=None,
           appearance=None):
    """region_oracle.render with the appearance applied after the selection and the exclusion in both passes, so the edited
    coarse weights drive sample_pdf.  raw_* are the unedited network outputs."""
    from .dmnerf_oracle import _net_inputs, mlp_forward, sample_pdf, stratify
    from .region_oracle import _selected
    viewdirs = rays_d / torch.norm(rays_d, dim=-1, keepdim=True)
    if perturb > 0.0:
        z_coarse = stratify(z_coarse, t_rand)
    x, shp = _net_inputs(rays_o, rays_d, viewdirs, z_coarse)
    raw_c = mlp_forward(p_coarse, x).reshape(*shp, -1)
    rgb_c, w_c, depth_c, ins_c, acc_c = composite(raw_c, _selected(raw_c, keep, z_coarse, exclude), z_coarse, rays_d, appearance)
    z_mid = 0.5 * (z_coarse[..., 1:] + z_coarse[..., :-1])
    z_samples = sample_pdf(z_mid, w_c[..., 1:-1], n_importance, det=(perturb == 0.0), u=u).detach()
    z_fine, _ = torch.sort(torch.cat([z_coarse, z_samples], -1), -1)
    x, shp = _net_inputs(rays_o, rays_d, viewdirs, z_fine)
    raw_f = mlp_forward(p_fine, x).reshape(*shp, -1)
    rgb_f, w_f, depth_f, ins_f, acc_f = composite(raw_f, _selected(raw_f, keep, z_fine, exclude), z_fine, rays_d, appearance)
    return {"rgb_fine": rgb_f, "ins_fine": ins_f, "z_vals_fine": z_fine, "raw_fine": raw_f,
            "raw_coarse": raw_c, "rgb_coarse": rgb_c, "ins_coarse": ins_c, "z_vals_coarse": z_coarse,
            "depth_fine": depth_f, "depth_coarse": depth_c,
            "weights_coarse": w_c, "weights_fine": w_f, "acc_coarse": acc_c, "acc_fine": acc_f}


def render_on_depths(net_c, net_f, rays_o, rays_d, z_coarse, z_fine, fp32_inputs=True, keep=None, keep_all_ins=False,
                     exclude=None, appearance=None):
    """region_oracle.render_on_depths (teacher-forced on a kernel's own depths, each pass composited in fp64) with the
    appearance applied after the selection and the exclusion; the same keys."""
    from . import dmnerf_f16 as H
    from . import dmnerf_oracle as O
    from . import objects_oracle as OO
    from .region_oracle import _selected
    ro, rd = rays_o.double(), rays_d.double()
    viewdirs = rd / torch.norm(rd, dim=-1, keepdim=True)
    out = {}
    for tag, net, z in (("coarse", net_c, z_coarse), ("fine", net_f, z_fine)):
        if net is None:
            continue
        z = z.double()
        x = H.net_inputs_fp32(rays_o, rays_d, z) if fp32_inputs else O._net_inputs(ro, rd, viewdirs, z)[0]
        raw = net(x).double().reshape(z.shape[0], z.shape[1], -1)
        rgb, w, depth, ins, acc = composite(raw, _selected(raw, keep, z, exclude), z, rd, appearance, keep_all_ins)
        top2 = torch.topk(torch.sigmoid(raw[..., 4:]), 2, dim=-1).values
        out.update({"rgb_" + tag: rgb, "depth_" + tag: depth, "acc_" + tag: acc, "ins_" + tag: ins, "weights_" + tag: w,
                    "raw_" + tag: raw, "labels_" + tag: OO.object_labels(raw), "gap_" + tag: top2[..., 0] - top2[..., 1]})
    return out
