"""CPU oracle of object selection -- TEST INFRASTRUCTURE ONLY (same standing as oracle/dmnerf_oracle.py, whose restatement of the
original's dm_nerf it extends; the product package never imports it).

A selection keeps a set of object labels 0 .. ins_num.  Every network sample is labelled argmax(sigmoid(raw[..., 4:])), first
maximum (the original's exchanger rule, networks/manipulator.py:19-21); where that label is not kept the sample's density
raw[..., 3] is zeroed before the composite: relu(0) * dist = 0 gives alpha = 0, also on the 1e10 tail sample, and the rest of
the composite (networks/render.py:6-28) is unchanged.  oracle/make_golden_objects.py checks `render` bit for bit against the
original's unmodified dm_nerf with its networks' outputs edited this way."""
import torch

from oracle.dmnerf_oracle import _net_inputs, composite, mlp_forward, sample_pdf, stratify


def object_labels(raw):
    """Per-sample object label: argmax(sigmoid(raw[..., 4:])), first maximum (manipulator.py:19-21)."""
    return torch.argmax(torch.sigmoid(raw[..., 4:]), dim=-1)


def keep_table(words, n_labels):
    """The 4-word object mask -> bool [n_labels] (label k kept)."""
    return torch.tensor([bool((int(words[k >> 5]) >> (k & 31)) & 1) for k in range(n_labels)])


def select_objects(raw, keep):
    """raw[..., 3] (density) zeroed where the sample's label is not kept (keep: bool [ins_num + 1]); a new tensor."""
    kept = keep.to(raw.device)[object_labels(raw)]
    out = raw.clone()
    out[..., 3] = torch.where(kept, raw[..., 3], torch.zeros_like(raw[..., 3]))
    return out


def render(rays_o, rays_d, p_coarse, p_fine, z_coarse, keep, perturb=0.0, n_importance=128, t_rand=None, u=None):
    """dmnerf_oracle.render (dm_nerf(), networks/render.py:31-96) with the selection `keep` applied to both networks' outputs
    before their composites, so the selected coarse weights drive sample_pdf.  The returned raw_* are the unedited network
    outputs.  Inference only (no is_train slicing)."""
    viewdirs = rays_d / torch.norm(rays_d, dim=-1, keepdim=True)                    # :37
    if perturb > 0.0:
        z_coarse = stratify(z_coarse, t_rand)                                       # :40-47
    x, shp = _net_inputs(rays_o, rays_d, viewdirs, z_coarse)
    raw_c = mlp_forward(p_coarse, x).reshape(*shp, -1)                              # :60-61
    rgb_c, w_c, depth_c, ins_c, acc_c = composite(select_objects(raw_c, keep), z_coarse, rays_d)   # :63
    z_mid = 0.5 * (z_coarse[..., 1:] + z_coarse[..., :-1])                          # :66
    z_samples = sample_pdf(z_mid, w_c[..., 1:-1], n_importance, det=(perturb == 0.0), u=u).detach()  # :67-68
    z_fine, _ = torch.sort(torch.cat([z_coarse, z_samples], -1), -1)                # :70
    x, shp = _net_inputs(rays_o, rays_d, viewdirs, z_fine)
    raw_f = mlp_forward(p_fine, x).reshape(*shp, -1)                                # :82-83
    rgb_f, w_f, depth_f, ins_f, acc_f = composite(select_objects(raw_f, keep), z_fine, rays_d)     # :86
    return {"rgb_fine": rgb_f, "ins_fine": ins_f, "z_vals_fine": z_fine, "raw_fine": raw_f,
            "raw_coarse": raw_c, "rgb_coarse": rgb_c, "ins_coarse": ins_c, "z_vals_coarse": z_coarse,
            "depth_fine": depth_f, "depth_coarse": depth_c,
            "weights_coarse": w_c, "weights_fine": w_f, "acc_coarse": acc_c, "acc_fine": acc_f}
