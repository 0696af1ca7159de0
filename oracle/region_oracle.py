"""CPU oracle of region selection -- TEST INFRASTRUCTURE ONLY (the product package never imports it).

Restates DESIGN.md, "Region selection" in numpy fp32, one rounding per operation (numpy float32 arrays neither contract nor
widen), so that it reproduces the kernels bit for bit:
  voxel map    [M | c] = fp32(inv(A)), fp32(-inv(A) b) from objects.grid_affine in fp64;
  sample point p = o + d z per axis (fp32 product, then fp32 sum), as the network prologue;
  voxel        u_a = ((M_a0 p0 + M_a1 p1) + M_a2 p2) + c_a, i_a = rint(u_a) (half to even), inside when 0 <= i_a <= dim - 1;
  bit          bit v & 31 of word v >> 5, v = (i0 dim + i1) dim + i2;
  rule         a sample with label l in `applies` is excluded inside the grid where its bit is 0, outside it unless outside_keep.
The builders: pack is a table look-up over a component id grid, dilate is scipy.ndimage.binary_dilation with the 6- or 26-
neighbourhood, `r` iterations (r = 0: none) and a zero border.
The renders: `render` is objects_oracle.render and `render_on_depths` is dmnerf_f16.render_on_depths, each with an optional
per-sample exclusion (a region's rule, `exclusion`) applied after the label selection; without one they return what those do."""
import numpy as np
import torch


def voxel_map(A, b):
    """[M | c] float32 [3, 4] from the fp64 grid affine p = A idx + b."""
    A, b = np.asarray(A, dtype=np.float64), np.asarray(b, dtype=np.float64)
    M = np.linalg.inv(A)
    return np.concatenate([M, (-M @ b)[:, None]], 1).astype(np.float32)


def voxel_of(vmap, pts):
    """rint(u) float32 [n, 3] of the points pts [n, 3] (float32) under the voxel map: the kernels' arithmetic."""
    f = np.float32
    m = np.asarray(vmap, dtype=f).reshape(3, 4)
    p = np.asarray(pts, dtype=f).reshape(-1, 3)
    with np.errstate(invalid="ignore", over="ignore"):
        u = np.stack([((m[a, 0] * p[:, 0] + m[a, 1] * p[:, 1]) + m[a, 2] * p[:, 2]) + m[a, 3] for a in range(3)], -1)
        return np.rint(u)


def lookup(vmap, bits, dim, pts):
    """Per point: 1 / 0 inside the grid (its bit), -1 outside (NaN and inf included) -> int8 [n]."""
    i = voxel_of(vmap, pts)
    with np.errstate(invalid="ignore"):
        inside = np.all((i >= 0) & (i <= dim - 1), axis=-1)
    out = np.full(i.shape[0], -1, dtype=np.int8)
    ii = i[inside].astype(np.int64)
    v = (ii[:, 0] * dim + ii[:, 1]) * dim + ii[:, 2]
    words = np.asarray(bits).view(np.uint32)
    out[inside] = ((words[v >> 5] >> (v & 31).astype(np.uint32)) & 1).astype(np.int8)
    return out


def contains(vmap, bits, dim, pts):
    """dmnerf_region_contains: inside the grid and bit set -> bool [n]."""
    return lookup(vmap, bits, dim, pts) == 1


def pack(mask):
    """Packed words (uint32, ceil(n / 32)) of a boolean grid in C order; the tail zero."""
    flat = np.asarray(mask, dtype=bool).reshape(-1)
    n = flat.size
    padded = np.zeros((n + 31) // 32 * 32, dtype=np.uint64)
    padded[:n] = flat
    return (padded.reshape(-1, 32) << np.arange(32, dtype=np.uint64)).sum(1).astype(np.uint32)


def unpack(words, dim):
    """The boolean grid [dim]^3 of packed words."""
    w = np.asarray(words).view(np.uint32).astype(np.uint64)
    bits = ((w[:, None] >> np.arange(32, dtype=np.uint64)) & 1).astype(bool).reshape(-1)
    return bits[:dim ** 3].reshape(dim, dim, dim)


def pack_ids(ids, chosen):
    """pack of the points whose id (int32 grid, -1 = none) is in `chosen`."""
    ids = np.asarray(ids)
    return pack(np.isin(ids, np.asarray(sorted(chosen), dtype=np.int64)) & (ids >= 0))


def dilate(mask, r, connectivity=26):
    """scipy's binary dilation, r steps (r = 0: the mask itself), zero border."""
    from scipy import ndimage
    mask = np.asarray(mask, dtype=bool)
    if r == 0:
        return mask.copy()
    st = ndimage.generate_binary_structure(3, 1 if connectivity == 6 else 3)
    return ndimage.binary_dilation(mask, st, iterations=r, border_value=0)


def sample_points(rays_o, rays_d, z):
    """p = o + d z per sample in fp32 (the network prologue's expression) -> [N, S, 3]."""
    f = np.float32
    o = np.asarray(rays_o, dtype=f)[:, None, :]
    d = np.asarray(rays_d, dtype=f)[:, None, :]
    return o + d * np.asarray(z, dtype=f)[..., None]


def exclusion(vmap, bits, dim, applies, outside_keep, rays_o, rays_d):
    """The region rule as a per-sample exclusion for objects_oracle.render / dmnerf_f16.render_on_depths: a callable
    (z [N, S], labels [N, S]) -> bool [N, S], True where the region gives the sample alpha = 0."""
    applies = [int(w) for w in applies]

    def excluded(z, labels):
        z = z.detach().cpu().float().numpy() if torch.is_tensor(z) else np.asarray(z, dtype=np.float32)
        lab = labels.detach().cpu().numpy() if torch.is_tensor(labels) else np.asarray(labels)
        n, s = z.shape
        b = lookup(vmap, bits, dim, sample_points(rays_o, rays_d, z).reshape(-1, 3)).reshape(n, s)
        on = np.array([(applies[k >> 5] >> (k & 31)) & 1 for k in range(128)], dtype=bool)[lab]
        return torch.from_numpy(on & ((b == 0) | ((b < 0) & (not outside_keep))))
    return excluded


def exclude_samples(raw, excluded):
    """raw[..., 3] (density) zeroed where excluded (bool [N, S]): relu(0) * dist = 0 gives alpha = 0; a new tensor."""
    out = raw.clone()
    out[..., 3] = torch.where(excluded.to(raw.device), torch.zeros_like(raw[..., 3]), raw[..., 3])
    return out


def _selected(raw, keep, z, exclude):
    """raw with the label selection keep (bool [ins_num + 1], or None) and then the exclusion applied."""
    from . import objects_oracle as OO
    sel = raw if keep is None else OO.select_objects(raw, keep)
    return sel if exclude is None else exclude_samples(sel, exclude(z, OO.object_labels(raw)))


def render(rays_o, rays_d, p_coarse, p_fine, z_coarse, keep, perturb=0.0, n_importance=128, t_rand=None, u=None, exclude=None):
    """objects_oracle.render (dm_nerf(), networks/render.py:31-96, with the selection `keep`) with the exclusion `exclude`
    ((z [N, S], labels [N, S]) -> bool [N, S], or None) applied after the selection in both passes, so the cleaned coarse
    weights drive sample_pdf.  raw_* are the unedited network outputs."""
    from .dmnerf_oracle import _net_inputs, composite, mlp_forward, sample_pdf, stratify
    viewdirs = rays_d / torch.norm(rays_d, dim=-1, keepdim=True)                    # :37
    if perturb > 0.0:
        z_coarse = stratify(z_coarse, t_rand)                                       # :40-47
    x, shp = _net_inputs(rays_o, rays_d, viewdirs, z_coarse)
    raw_c = mlp_forward(p_coarse, x).reshape(*shp, -1)                              # :60-61
    rgb_c, w_c, depth_c, ins_c, acc_c = composite(_selected(raw_c, keep, z_coarse, exclude), z_coarse, rays_d)   # :63
    z_mid = 0.5 * (z_coarse[..., 1:] + z_coarse[..., :-1])                          # :66
    z_samples = sample_pdf(z_mid, w_c[..., 1:-1], n_importance, det=(perturb == 0.0), u=u).detach()  # :67-68
    z_fine, _ = torch.sort(torch.cat([z_coarse, z_samples], -1), -1)                # :70
    x, shp = _net_inputs(rays_o, rays_d, viewdirs, z_fine)
    raw_f = mlp_forward(p_fine, x).reshape(*shp, -1)                                # :82-83
    rgb_f, w_f, depth_f, ins_f, acc_f = composite(_selected(raw_f, keep, z_fine, exclude), z_fine, rays_d)     # :86
    return {"rgb_fine": rgb_f, "ins_fine": ins_f, "z_vals_fine": z_fine, "raw_fine": raw_f,
            "raw_coarse": raw_c, "rgb_coarse": rgb_c, "ins_coarse": ins_c, "z_vals_coarse": z_coarse,
            "depth_fine": depth_f, "depth_coarse": depth_c,
            "weights_coarse": w_c, "weights_fine": w_f, "acc_coarse": acc_c, "acc_fine": acc_f}


def render_on_depths(net_c, net_f, rays_o, rays_d, z_coarse, z_fine, fp32_inputs=True, keep=None, keep_all_ins=False,
                     exclude=None):
    """dmnerf_f16.render_on_depths (the teacher-forced render on a kernel's own depths, each pass composited in fp64) with the
    exclusion `exclude` applied after the selection; the same keys: rgb_p, depth_p, acc_p, ins_p, weights_p, raw_p
    (unselected), labels_p and gap_p for p in (coarse, fine)."""
    from . import dmnerf_f16 as H
    from . import dmnerf_oracle as O
    from . import objects_oracle as OO
    ro, rd = rays_o.double(), rays_d.double()
    viewdirs = rd / torch.norm(rd, dim=-1, keepdim=True)
    out = {}
    for tag, net, z in (("coarse", net_c, z_coarse), ("fine", net_f, z_fine)):
        if net is None:
            continue
        z = z.double()
        x = H.net_inputs_fp32(rays_o, rays_d, z) if fp32_inputs else O._net_inputs(ro, rd, viewdirs, z)[0]
        raw = net(x).double().reshape(z.shape[0], z.shape[1], -1)
        rgb, w, depth, ins, acc = O.composite(_selected(raw, keep, z, exclude), z, rd, keep_all_ins=keep_all_ins)
        top2 = torch.topk(torch.sigmoid(raw[..., 4:]), 2, dim=-1).values
        out.update({"rgb_" + tag: rgb, "depth_" + tag: depth, "acc_" + tag: acc, "ins_" + tag: ins, "weights_" + tag: w,
                    "raw_" + tag: raw, "labels_" + tag: OO.object_labels(raw), "gap_" + tag: top2[..., 0] - top2[..., 1]})
    return out
