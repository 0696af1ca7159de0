"""CPU oracle for the DM-NeRF per-ray render path -- TEST INFRASTRUCTURE ONLY.

This file is a functional, dtype-generic restatement (torch CPU ops, fp32 by default, fp64 for the
noise-floor twin) of the reference algorithm in /root/reference/networks/{render,dm_nerf,helpers}.py.
It exists only to check the CUDA path: only tests/, __graft_entry__.smoke() and the cpu_baseline /
--impl reference legs of bench.py may import it.  The product package (dm-nerf_b200/) never does.

Parity pinning: the reference ships NO tests, golden vectors or checkpoints (SURVEY.md section 4), so
the pin is the reference code itself: oracle/make_golden.py imports the unmodified reference from
/root/reference in the build container, checks every function below against it on seeded inputs
and writes the reference's outputs to tests/golden/*.npz.  tests/test_oracle.py re-checks this oracle against
those committed fixtures wherever the tests run.

Every function cites the reference lines it restates.  Weights are passed as a plain dict keyed by
the reference state_dict names (networks/dm_nerf.py:65-78).
"""
import numpy as np
import torch
import torch.nn.functional as F

SKIPS = (4,)
N_TRUNK = 8


def embed(x, n_freqs):
    """Positional encoding, reference networks/dm_nerf.py:13-38 with get_embedder's kwargs (:45-52):
    [x, sin(2^0 x), cos(2^0 x), ..., sin(2^(L-1) x), cos(2^(L-1) x)]; frequencies are exact powers of two."""
    parts = [x]
    for k in range(n_freqs):
        xf = x * float(2 ** k)
        parts.append(torch.sin(xf))
        parts.append(torch.cos(xf))
    return torch.cat(parts, -1)


def _lin(p, name, x):
    return F.linear(x, p[name + ".weight"], p[name + ".bias"])


def mlp_forward(p, x, ch_pts=63, ch_views=27):
    """DM_NeRF.forward, reference networks/dm_nerf.py:80-106. x [M, 63+27] -> [M, 3+1+ins_num+1]."""
    pts, dirs = x[..., :ch_pts], x[..., ch_pts:ch_pts + ch_views]
    h = pts
    for i in range(N_TRUNK):
        h = torch.relu(_lin(p, "mlps.%d" % i, h))                                  # :84-85
        if i in SKIPS:
            h = torch.cat([h, pts], -1)                                            # :86-87  order [h, pts]
    rgb_f = _lin(p, "rgb_feature_linear", h)                                        # :89 (no activation)
    rgb_f = torch.relu(_lin(p, "rgb_feature_linears.0", torch.cat([rgb_f, dirs], -1)))   # :90-93
    ins_f = _lin(p, "ins_feature_linear", h.detach())                               # :95-96 (h is detached)
    ins_f = torch.relu(_lin(p, "ins_feature_linears.0", ins_f))                     # :97-99
    density = _lin(p, "density_linear", h)                                          # :101
    rgb = _lin(p, "rgb_linear", rgb_f)                                              # :102
    ins = _lin(p, "ins_linear", ins_f)                                              # :103
    return torch.cat([rgb, density, ins], -1)                                       # :105


def composite(raw, z_vals, rays_d, keep_all_ins=False):
    """render_train, reference networks/render.py:6-28 (keep_all_ins=True gives manipulator_render,
    networks/manipulator.py:86-105).  Returns rgb_map, weights, depth_map, ins_map, acc_map."""
    dists = z_vals[..., 1:] - z_vals[..., :-1]
    tail = torch.full_like(dists[..., :1], 1e10)                                    # :10
    dists = torch.cat([dists, tail], -1)
    dists = dists * torch.norm(rays_d[..., None, :], dim=-1)                        # :12
    rgb = torch.sigmoid(raw[..., :3])                                               # :14
    alpha = 1.0 - torch.exp(-torch.relu(raw[..., 3]) * dists)                       # :7,16
    ones = torch.ones_like(alpha[..., :1])
    trans = torch.cumprod(torch.cat([ones, 1.0 - alpha + 1e-10], -1), -1)[..., :-1]  # :18
    weights = alpha * trans
    rgb_map = torch.sum(weights[..., None] * rgb, -2)                               # :19
    depth_map = torch.sum(weights * z_vals, -1)                                     # :20
    w_ins = weights if keep_all_ins else weights.detach()                           # :22-23 (manipulator.py:100 keeps grad)
    ins_map = torch.sigmoid(torch.sum(w_ins[..., None] * raw[..., 4:], -2))         # :24-25
    if not keep_all_ins:
        ins_map = ins_map[..., :-1]                                                 # :26
    acc_map = torch.sum(weights, -1)          # not in the reference; SURVEY.md name-mapping table
    return rgb_map, weights, depth_map, ins_map, acc_map


def sample_pdf(bins, weights, n_samples, det=False, u=None):
    """Inverse-CDF sampling, reference networks/helpers.py:123-155.  `u` replaces the reference's
    internal torch.rand draw (:135) so the caller controls the random stream."""
    weights = weights + 1e-5                                                        # :125
    pdf = weights / torch.sum(weights, -1, keepdim=True)
    cdf = torch.cumsum(pdf, -1)
    cdf = torch.cat([torch.zeros_like(cdf[..., :1]), cdf], -1)                      # :128
    if det:
        u = torch.linspace(0.0, 1.0, steps=n_samples, dtype=bins.dtype)             # :132
        u = u.expand(list(cdf.shape[:-1]) + [n_samples])
    return _inverse_cdf(bins, cdf, u)


def warp_cdf(weights):
    """The CDF of sample_pdf (helpers.py:125-128) in fp32, summed in the order of the library's one-warp samplers (ray_build_cdf,
    dm-nerf_b200/csrc/ray_ops.cuh): lane l (of 32) adds w[l], w[l + 32], ... in turn, a butterfly over the lanes gives the total,
    and each 32-wide chunk of the pdf is a Hillis-Steele inclusive scan added to the running carry.  The reference's CPU cumsum
    accumulates in fp64 instead; the two differ in the last bits, which moves samples where the inverse CDF is ill-conditioned.
    weights [N, B - 1] -> cdf [N, B]."""
    w = weights.float() + 1e-5                                                      # :125
    n, nw = w.shape
    chunks = (nw + 31) // 32
    lanes = torch.zeros(n, chunks * 32)
    lanes[:, :nw] = w
    lanes = lanes.reshape(n, chunks, 32)
    total = torch.zeros(n, 32)
    for c in range(chunks):
        total = total + lanes[:, c]
    for d in (16, 8, 4, 2, 1):
        total = total + total[:, torch.arange(32) ^ d]
    pdf = lanes / total[:, :1, None]
    cdf, carry = [torch.zeros(n, 1)], torch.zeros(n)
    for c in range(chunks):
        v = pdf[:, c]
        for d in (1, 2, 4, 8, 16):
            v = torch.cat([v[:, :d], v[:, d:] + v[:, :-d]], -1)
        cdf.append(carry[:, None] + v)
        carry = carry + v[:, 31]
    return torch.cat(cdf, -1)[:, :nw + 1].contiguous()


def sample_pdf_warp(bins, weights, n_samples, det=False, u=None):
    """sample_pdf with the CDF of warp_cdf: the library's samplers' arithmetic, operation for operation."""
    cdf = warp_cdf(weights)
    if det:
        u = torch.linspace(0.0, 1.0, steps=n_samples).expand(cdf.shape[0], n_samples)
    return _inverse_cdf(bins.float(), cdf, u.float())


def _inverse_cdf(bins, cdf, u):
    """helpers.py:137-153: the samples of u [N, n_samples] on the CDF cdf [N, B] over bins [N, B]."""
    u = u.contiguous()
    inds = torch.searchsorted(cdf, u, right=True)                                   # :139
    below = torch.clamp(inds - 1, min=0)
    above = torch.clamp(inds, max=cdf.shape[-1] - 1)
    cdf_b, cdf_a = torch.gather(cdf, -1, below), torch.gather(cdf, -1, above)
    bin_b, bin_a = torch.gather(bins, -1, below), torch.gather(bins, -1, above)
    denom = cdf_a - cdf_b
    denom = torch.where(denom < 1e-5, torch.ones_like(denom), denom)                # :151
    t = (u - cdf_b) / denom
    return bin_b + t * (bin_a - bin_b)                                              # :153


def sample_pdf_explained(bins, weights, n_samples, det, u, tol):
    """Bool [N, n_samples]: which samples of sample_pdf(bins, weights, n_samples, det, u) the inverse CDF itself makes
    ill-conditioned, so that an fp32 implementation may legitimately land more than `tol` away from the fp32 oracle there:
      (a) u within a few ulp of a CDF knot (searchsorted picks the neighbouring bin),
      (b) a 3e-7 perturbation of the CDF (2 ulp of a value in [0,1]) already moves the sample by more than half the tolerance
          (tiny denom = almost empty bin, helpers.py:150-152), or
      (c) the reference's own arithmetic in fp64 lands elsewhere too.
    A miss outside this mask is an arithmetic error of the implementation.  bins [N, B], weights [N, B - 1], u [N, n_samples] or
    None (det), tol: scalar or array broadcastable to [N, n_samples]."""
    bins, weights = bins.cpu(), weights.cpu()
    u = None if u is None else u.cpu()
    n = bins.shape[0]
    ref = sample_pdf(bins.float(), weights.float(), n_samples, det=det, u=None if u is None else u.float()).numpy()
    uu = (torch.linspace(0.0, 1.0, n_samples).expand(n, n_samples) if det else u).double()
    wd = weights.double() + 1e-5
    cdf = torch.cat([torch.zeros(n, 1, dtype=torch.float64), torch.cumsum(wd / wd.sum(-1, keepdim=True), -1)], -1)
    knot = (uu[..., None] - cdf[:, None, :]).abs().min(-1).values.numpy() <= 4e-7                           # (a)
    inds = torch.searchsorted(cdf.float().contiguous(), uu.float().contiguous(), right=True)
    below, above = (inds - 1).clamp(min=0), inds.clamp(max=cdf.shape[-1] - 1)
    denom = (torch.gather(cdf, -1, above) - torch.gather(cdf, -1, below))
    width = (torch.gather(bins.double(), -1, above) - torch.gather(bins.double(), -1, below)).abs()
    cond = (width * 3e-7 / denom.clamp(min=1e-12)).numpy() > 0.5 * tol                                        # (b)
    twin = sample_pdf(bins.double(), weights.double(), n_samples, det=det, u=None if u is None else u.double()).numpy()
    twin_bad = np.abs(twin - ref) > tol                                                                       # (c)
    return knot | cond | twin_bad


def hier_sample(z_c, w_c, n_importance, det, u=None):
    """The fine depths of reference networks/render.py:66-70 from given coarse depths z_c [N, S] and weights w_c [N, S]:
    sample_pdf on the mid-points with weights[1:-1], then sort(cat(coarse, samples)).  NaN samples sort last, as torch.sort
    puts them."""
    z_mid = 0.5 * (z_c[..., 1:] + z_c[..., :-1])                                    # :66
    z_samples = sample_pdf(z_mid, w_c[..., 1:-1], n_importance, det=det, u=u).detach()   # :67-68
    return torch.sort(torch.cat([z_c, z_samples], -1), -1)[0]                       # :70


def z_val_sample(n_rays, near, far, n_samples, dtype=torch.float32):
    """reference networks/helpers.py:114-119: near + linspace(0,1,S) * (far - near), expanded to N rows."""
    t = torch.linspace(0.0, 1.0, steps=n_samples, dtype=dtype)
    near_t = near * torch.ones((n_rays, 1), dtype=dtype)
    far_t = far * torch.ones((n_rays, 1), dtype=dtype)
    return (near_t + t * (far_t - near_t)).expand(n_rays, n_samples)


def get_rays_k(H, W, K, c2w):
    """reference networks/helpers.py:50-61."""
    i, j = torch.meshgrid(torch.linspace(0, W - 1, W), torch.linspace(0, H - 1, H), indexing="ij")
    i, j = i.t(), j.t()
    dirs = torch.stack([(i - K[0, 2]) / K[0, 0], (j - K[1, 2]) / K[1, 1], K[2, 2] * torch.ones_like(i)], -1)
    rays_d = torch.sum(dirs[..., None, :] * c2w[:3, :3], -1)
    rays_o = c2w[:3, -1].expand(rays_d.shape)
    return rays_o, rays_d


def stratify(z, t_rand):
    """Stratified jitter, reference networks/render.py:40-47."""
    mids = 0.5 * (z[..., 1:] + z[..., :-1])
    upper = torch.cat([mids, z[..., -1:]], -1)
    lower = torch.cat([z[..., :1], mids], -1)
    return lower + (upper - lower) * t_rand


def _net_inputs(rays_o, rays_d, viewdirs, z):
    pts = rays_o[..., None, :] + rays_d[..., None, :] * z[..., :, None]             # render.py:49,71
    flat = pts.reshape(-1, 3)
    dirs = viewdirs[:, None].expand(pts.shape).reshape(-1, 3)                       # render.py:55-56
    return torch.cat([embed(flat, 10), embed(dirs, 4)], -1), pts.shape[:-1]          # render.py:54-58


def render(rays_o, rays_d, p_coarse, p_fine, z_coarse, perturb=0.0, n_importance=128,
           t_rand=None, u=None, is_train=False, n_ins=None):
    """dm_nerf(), reference networks/render.py:31-96.  t_rand [N,S] and u [N,I] are the two uniform
    draws the reference takes from torch.rand (render.py:46, helpers.py:135), in that order."""
    viewdirs = rays_d / torch.norm(rays_d, dim=-1, keepdim=True)                    # :37
    if perturb > 0.0:
        z_coarse = stratify(z_coarse, t_rand)                                       # :40-47
    x, shp = _net_inputs(rays_o, rays_d, viewdirs, z_coarse)
    raw_c = mlp_forward(p_coarse, x).reshape(*shp, -1)                              # :60-61
    rgb_c, w_c, depth_c, ins_c, acc_c = composite(raw_c, z_coarse, rays_d)           # :63
    z_mid = 0.5 * (z_coarse[..., 1:] + z_coarse[..., :-1])                          # :66
    z_samples = sample_pdf(z_mid, w_c[..., 1:-1], n_importance, det=(perturb == 0.0), u=u).detach()  # :67-68
    z_fine, _ = torch.sort(torch.cat([z_coarse, z_samples], -1), -1)                # :70
    x, shp = _net_inputs(rays_o, rays_d, viewdirs, z_fine)
    raw_f = mlp_forward(p_fine, x).reshape(*shp, -1)                                # :82-83
    rgb_f, w_f, depth_f, ins_f, acc_f = composite(raw_f, z_fine, rays_d)             # :86
    if is_train and n_ins is not None:
        ins_f, ins_c = ins_f[-n_ins:], ins_c[-n_ins:]                               # :88-90
    return {"rgb_fine": rgb_f, "ins_fine": ins_f, "z_vals_fine": z_fine, "raw_fine": raw_f,
            "raw_coarse": raw_c, "rgb_coarse": rgb_c, "ins_coarse": ins_c, "z_vals_coarse": z_coarse,
            "depth_fine": depth_f, "depth_coarse": depth_c,
            # extras (not in the reference dict): weights and acc maps
            "weights_coarse": w_c, "weights_fine": w_f, "acc_coarse": acc_c, "acc_fine": acc_f}


def to_torch(weights_np, dtype=torch.float32):
    return {k: torch.from_numpy(v).to(dtype) for k, v in weights_np.items()}


def train_loss(out, target_rgb):
    """Scalar loss used for the training-step parity case C4 (SURVEY.md 8d): the rgb MSE terms of
    train_dmsr.py:35-37 plus mean(ins) stand-ins for the instance terms (the Hungarian loss itself is
    out of scope)."""
    return (((out["rgb_coarse"] - target_rgb) ** 2).mean() + ((out["rgb_fine"] - target_rgb) ** 2).mean()
            + out["ins_coarse"].mean() + out["ins_fine"].mean())


def emptiness_penalizer(raw, z_vals, depths, rays_d, tolerance, deta_w):
    """"Emptiness" regulariser on the per-sample object logits, reference networks/penalizer.py:5-55.
    raw [N,S,4+K], z_vals [N,S], depths [N,1] (already detached, penalizer.py:59), rays_d [N,3] -> loss tensor of shape [1].
    In front of the surface (more than `tolerance` before the rendered depth) every sample should be "no object" (last class),
    weighted by 1 - gaussian(distance to the surface); inside the +-tolerance shell the last class is pushed to 0, weighted by
    the gaussian.  Both terms are masked means (penalizer.py:41-42, 52)."""
    sigma_h = torch.Tensor([0.4])                                                   # :10
    sigma_w = torch.Tensor([deta_w])
    two_pi_root = torch.sqrt(torch.Tensor([2 * np.pi]))

    def gaussian(delta):                                                            # :7-8
        return torch.exp(-(delta ** 2) / (2 * (sigma_w ** 2))) / (sigma_h * two_pi_root) + 1e-8

    norm = torch.norm(rays_d[..., None, :], dim=-1)                                 # :13   [N,1]
    front = (depths - tolerance) * norm                                             # :14,16
    back = (depths + tolerance) * norm                                              # :15,17
    surface = depths * norm                                                         # :18
    pos = z_vals * norm                                                             # :19
    g = gaussian(surface - pos)                                                     # :22-23
    air = 1 - g                                                                     # :24
    m_before = (pos < front).type(torch.float32)                                    # :27
    m_after = (pos > back).type(torch.float32)                                      # :28
    m_middle = 1 - (m_after + m_before)                                             # :29
    pred = torch.sigmoid(raw[..., 4:])                                              # :32-33
    gt = torch.zeros_like(pred)
    gt[..., -1] = 1                                                                 # :37-38
    l_before = -gt * torch.log(pred + 1e-8) - (1 - gt) * torch.log(1 - pred + 1e-8)  # :39
    l_before = l_before * (air * m_before)[..., None]                               # :40-41
    l_before = torch.sum(l_before) / (pred.shape[-1] * torch.maximum(torch.sum(m_before), torch.tensor([1e-8])))   # :42-43
    last = pred[..., -1]                                                            # :46
    gt_mid = torch.zeros_like(last)
    l_mid = -gt_mid * torch.log(last + 1e-8) - (1 - gt_mid) * torch.log(1 - last + 1e-8)   # :48-49
    l_mid = l_mid * (g * m_middle)                                                  # :50-51
    l_mid = torch.sum(l_mid) / torch.maximum(torch.sum(m_middle), torch.tensor([1e-8]))    # :52
    return l_before + l_mid                                                         # :53


def ins_penalizer(raw, z_vals, depth, rays_d, tolerance, deta_w):
    """networks/penalizer.py:58-62 (args.tolerance / args.deta_w passed explicitly)."""
    return emptiness_penalizer(raw, z_vals, depth[..., None].detach(), rays_d, tolerance, deta_w)


# ------------------------------------------------------------------------------------------------------------------
# Object manipulation at render time (SURVEY.md section 8, row f3): reference networks/manipulator.py:18-205.
# ------------------------------------------------------------------------------------------------------------------
def manipulator_nerf(p, rays, z_vals=None, n_samples=None, near=None, far=None):
    """One network evaluated along the rays at given (or freshly spaced) depths, manipulator.py:108-134.
    Note the depth formula near*(1-t) + far*t (:119), which differs from z_val_sample's in the last bits."""
    rays_o, rays_d = rays
    viewdirs = rays_d / torch.norm(rays_d, dim=-1, keepdim=True)                      # :110-112
    n_rays = rays_d.shape[0]
    if z_vals is None:
        near_, far_ = near * torch.ones(size=(n_rays, 1)), far * torch.ones(size=(n_rays, 1))
        t_vals = torch.linspace(0., 1., steps=n_samples)
        z_vals = (near_ * (1. - t_vals) + far_ * t_vals).expand([n_rays, n_samples])   # :117-120
    pts = rays_o[..., None, :] + rays_d[..., None, :] * z_vals[..., :, None]          # :122
    x = torch.cat([embed(pts.reshape(-1, 3), 10), embed(viewdirs[:, None].expand(pts.shape).reshape(-1, 3), 4)], -1)
    raw = mlp_forward(p, x)                                                          # :131
    return raw.reshape(list(pts.shape[:-1]) + [raw.shape[-1]]), z_vals


def manipulator_render(raw, z_vals, rays_d):
    """manipulator.py:86-105: the composite without the detach and with every instance channel kept."""
    rgb, weights, depth, ins, _ = composite(raw, z_vals, rays_d, keep_all_ins=True)
    return rgb, weights, depth, ins


def exchanger(ori_raw, tar_raws, ori_raw_pred, tar_raw_preds, move_labels):
    """Per-sample swap of network outputs between the original and the transformed rays, manipulator.py:18-83.
    Returns (edited ori_raw, tar_raws, per-sample label of the original, per-sample label of the last target)."""
    ori_raw = ori_raw.clone()
    ori_label = torch.argmax(torch.sigmoid(ori_raw[..., 4:]), dim=-1)                 # :19-21
    ori_acc = torch.argmax(torch.sigmoid(ori_raw_pred[..., :-1]), dim=-1)             # :23-25 (last = "empty" class dropped)
    ori_acc = ori_acc[:, None].expand_as(ori_label)                                   # :26
    tar_label = None
    for idx, mv in enumerate(move_labels):
        tar_raw = tar_raws[idx]
        ori_label = torch.where((ori_label == mv) & (ori_acc != mv), ori_acc, ori_label)     # :33-36 occluder in front
        fillings = (ori_acc == mv) & (ori_label != mv)                                # :40-42
        tar_label = torch.argmax(torch.sigmoid(tar_raw[..., 4:]), dim=-1)             # :45-47
        tar_acc = torch.argmax(torch.sigmoid(tar_raw_preds[idx][..., :-1]), dim=-1)[:, None].expand_as(tar_label)   # :50-53
        tar_label = torch.where((tar_label == mv) & (tar_acc != mv), tar_acc, tar_label)     # :57-60
        code = (tar_label == mv).long() + 2 * (ori_label == mv).long()                # :64-69: 0 none, 1 target only, 2 original only, 3 both
        take = (code == 1) | (code == 3)                                              # :71-75  exchange
        wipe = code == 2                                                              #         eliminate
        ori_raw = torch.where(fillings[..., None], tar_raw, ori_raw)                  # :78
        ori_raw = torch.where(take[..., None], tar_raw, ori_raw)                      # :81
        ori_raw = torch.where(wipe[..., None], ori_raw * 0, ori_raw)                  # :82
    return ori_raw, tar_raws, ori_label, tar_label


def manipulator(p_coarse, p_fine, ori_rays, f_tar_rays, n_samples, n_importance, near, far, target_labels, us=None):
    """Whole edit-time pipeline for one chunk of rays, manipulator.py:137-205.  The reference calls sample_pdf without
    det=True, i.e. with torch.rand draws (helpers.py:135), in the order: original rays, each target, original again (step 2).
    `us` (a list of [N, n_importance] tensors consumed in that order) replaces the draws; None draws from torch's global
    generator exactly like the reference."""
    us = list(us) if us is not None else None

    def draw(bins, w):
        return sample_pdf(bins, w, n_importance, u=(us.pop(0) if us is not None else None))

    def fine_pass(rays, coarse_raw, coarse_z):
        _, w, _, _ = manipulator_render(coarse_raw, coarse_z, rays[1])
        mid = .5 * (coarse_z[..., 1:] + coarse_z[..., :-1])
        z_s = draw(mid, w[..., 1:-1])                                                 # :147-148 (random u)
        z_full, _ = torch.sort(torch.cat([coarse_z, z_s], -1), -1)
        raw_full, _ = manipulator_nerf(p_fine, rays, z_vals=z_full)
        _, _, _, ins_acc = manipulator_render(raw_full, z_full, rays[1])
        return z_s, ins_acc

    ori_raw, ori_z = manipulator_nerf(p_coarse, ori_rays, None, n_samples, near, far)   # :140-141
    _, ori_ins_acc = fine_pass(ori_rays, ori_raw, ori_z)                              # :144-152
    tar_raws, tar_zs, tar_samples, tar_accs = [], [], [], []
    tar_rgb = None
    for tar_rays in f_tar_rays:                                                       # :155-176
        t_raw, t_z = manipulator_nerf(p_coarse, tar_rays, None, n_samples, near, far)
        tar_rgb, _, _, _ = manipulator_render(t_raw, t_z, tar_rays[1])
        z_s, acc = fine_pass(tar_rays, t_raw, t_z)
        tar_raws.append(t_raw); tar_zs.append(t_z); tar_samples.append(z_s); tar_accs.append(acc)
    ori_raw, _, _, _ = exchanger(ori_raw, tar_raws, ori_ins_acc, tar_accs, target_labels)    # :179
    _, ori_w, _, _ = manipulator_render(ori_raw, ori_z, ori_rays[1])                 # :183
    mid = .5 * (ori_z[..., 1:] + ori_z[..., :-1])
    ori_samples = draw(mid, ori_w[..., 1:-1])                                         # :186-187
    all_tar = torch.cat(tar_samples, -1)                                              # :190
    ori_z2, _ = torch.sort(torch.cat([ori_z, ori_samples, all_tar], -1), -1)          # :191
    ori_raw2 = None
    for idx, tar_rays in enumerate(f_tar_rays):                                       # :192-199
        ori_raw2, _ = manipulator_nerf(p_fine, ori_rays, z_vals=ori_z2)
        t_z2, _ = torch.sort(torch.cat([tar_zs[idx], ori_samples, all_tar], -1), -1)
        tar_raws[idx], _ = manipulator_nerf(p_fine, tar_rays, z_vals=t_z2)
    ori_raw2, _, _, _ = exchanger(ori_raw2, tar_raws, ori_ins_acc, tar_accs, target_labels)   # :201
    final_rgb, _, _, final_ins = manipulator_render(ori_raw2, ori_z2, ori_rays[1])    # :203
    return final_rgb, final_ins, tar_rgb, tar_accs[-1]


def hungarian(pred_ins, gt_ins, valid_ins_num, ins_num):
    """Matching, reference networks/evaluator.py:41-74.  pred_ins, gt_ins [N, ins_num] -> cost_ce, cost_siou
    [ins_num, ins_num] (row = ground-truth object, column = prediction channel), order_row, order_col."""
    from scipy.optimize import linear_sum_assignment
    pred = pred_ins.permute([1, 0])[None, :, :]                                    # :52-55
    gt = gt_ins.permute([1, 0])[:, None, :]
    cost_ce = torch.mean(-gt * torch.log(pred + 1e-8) - (1 - gt) * torch.log(1 - pred + 1e-8), dim=-1)   # :57
    tp = torch.sum(pred * gt, dim=-1)                                              # :60-64
    fp = torch.sum(pred, dim=-1) - tp
    fn = torch.sum(gt, dim=-1) - tp
    cost_siou = 1.0 - tp / (tp + fp + fn + 1e-6)
    with torch.no_grad():                                                          # reorder, :42-50
        scores = (cost_ce + cost_siou)[:valid_ins_num].cpu().numpy()
        row_ind, col_ind = linear_sum_assignment(scores)
        if ins_num - valid_ins_num > 0:
            unmapped = np.array(list(set(range(ins_num)) - set(col_ind)))
            col_ind = np.concatenate([col_ind, unmapped])
    return cost_ce, cost_siou, row_ind, col_ind


def ins_criterion(pred_ins, gt_labels, ins_num):
    """Hungarian-matched instance loss, reference networks/evaluator.py:19-37.  Returns (sum, valid_ce, invalid_ce, valid_siou)."""
    valid = torch.unique(gt_labels)                                                # :21
    gt_ins = torch.zeros(size=(gt_labels.shape[0], ins_num), dtype=pred_ins.dtype)
    n_valid = len(valid)
    gt_ins[..., :n_valid] = F.one_hot(gt_labels.long())[..., valid.long()].to(pred_ins.dtype)   # :25
    cost_ce, cost_siou, order_row, order_col = hungarian(pred_ins, gt_ins, n_valid, ins_num)
    valid_ce = torch.mean(cost_ce[order_row, order_col[:n_valid]])                 # :28
    if not (len(order_col) == n_valid):
        invalid_ce = torch.mean(pred_ins[:, order_col[n_valid:]])                  # :31
    else:
        invalid_ce = torch.tensor([0])
    valid_siou = torch.mean(cost_siou[order_row, order_col[:n_valid]])             # :34
    return valid_ce + invalid_ce + valid_siou, valid_ce, invalid_ce, valid_siou
