"""fp16-operand restatement of the DM_NeRF network -- TEST INFRASTRUCTURE ONLY.

The arithmetic of the fp16 preview network (DMNERF_IMPL_UMMA_F16, mlp_f16_kernel): every tensor-core GEMM takes fp16
operands and accumulates exactly (fp64 here; an fp16 x fp16 product is exact in fp32, so only the summation order differs
from the kernel's fp32 accumulator), biases are added after the sum.  Like the kernel:
  * every layer input that goes through the tensor core is rounded to fp16: the embeddings and the stored activations;
  * rgb_feature_linear / ins_feature_linear are folded into the layer after them in fp64 and rounded to fp32 (the fold
    buffer the exact pack also uses), then rounded to fp16 once;
  * density_linear and rgb_linear stay fp32 dot products on the unrounded fp32 activation (CUDA cores in the kernel).
It is the close yardstick for the fp16 kernel; the fp64 oracle (dmnerf_oracle.mlp_forward in float64) is the outer one.
"""
import torch

from . import dmnerf_oracle as O


def _h(t):
    """Round to fp16, continue in fp64."""
    return t.to(torch.float16).to(torch.float64)


def _gemm(a16, w, b):
    return a16 @ _h(w).t() + b


def folded_heads(p):
    """The kernel's folded head layers: (W_rgb [128, 283], b_rgb [128], W_ins [128, 256], b_ins [128]) in fp32, from the
    fp64 fold W' = W2 W1, b' = W2 b1 + b2 (the direction columns of rgb_feature_linears.0 are kept as they are)."""
    d = {k: v.to(torch.float64) for k, v in p.items()}
    w2r, w1r = d["rgb_feature_linears.0.weight"], d["rgb_feature_linear.weight"]
    w_rgb = torch.cat([w2r[:, :256] @ w1r, w2r[:, 256:]], 1)
    b_rgb = w2r[:, :256] @ d["rgb_feature_linear.bias"] + d["rgb_feature_linears.0.bias"]
    w2i, w1i = d["ins_feature_linears.0.weight"], d["ins_feature_linear.weight"]
    w_ins = w2i @ w1i
    b_ins = w2i @ d["ins_feature_linear.bias"] + d["ins_feature_linears.0.bias"]
    return tuple(t.to(torch.float32) for t in (w_rgb, b_rgb, w_ins, b_ins))


def mlp_forward_f16(p, x, ch_pts=63, ch_views=27):
    """DM_NeRF.forward with the fp16 kernel's arithmetic.  p: fp32 weights (state_dict names), x [M, 90] -> [M, C] float64."""
    d = {k: v.to(torch.float32) for k, v in p.items()}
    b = {k: v.to(torch.float64) for k, v in d.items()}
    x = x.to(torch.float32)
    pts16, dirs16 = _h(x[..., :ch_pts]), _h(x[..., ch_pts:ch_pts + ch_views])
    a16 = pts16
    h = None
    for i in range(O.N_TRUNK):
        # the kernel's accumulator is fp32: round every layer output to fp32 before the ReLU / the next fp16 rounding
        h = torch.relu(_gemm(a16, d["mlps.%d.weight" % i], b["mlps.%d.bias" % i]).to(torch.float32).to(torch.float64))
        a16 = _h(h)
        if i in O.SKIPS:
            a16 = torch.cat([a16, pts16], -1)
    w_rgb, b_rgb, w_ins, b_ins = folded_heads(d)
    density = h @ b["density_linear.weight"].t() + b["density_linear.bias"]
    rgb_h = torch.relu(_gemm(torch.cat([a16, dirs16], -1), w_rgb, b_rgb.to(torch.float64)).to(torch.float32).to(torch.float64))
    rgb = rgb_h @ b["rgb_linear.weight"].t() + b["rgb_linear.bias"]
    ins_h = torch.relu(_gemm(a16, w_ins, b_ins.to(torch.float64)).to(torch.float32).to(torch.float64))
    ins = _gemm(_h(ins_h), d["ins_linear.weight"], b["ins_linear.bias"])
    return torch.cat([rgb, density, ins], -1)


def render_f16(rays_o, rays_d, p_coarse, p_fine, z_coarse, n_importance=128):
    """Deterministic dm_nerf() (perturb = 0, oracle.render's pipeline) with both networks in fp16 arithmetic and the rest of
    the pipeline in fp64."""
    rays_o, rays_d, z_coarse = rays_o.double(), rays_d.double(), z_coarse.double()
    viewdirs = rays_d / torch.norm(rays_d, dim=-1, keepdim=True)
    x, shp = O._net_inputs(rays_o, rays_d, viewdirs, z_coarse)
    raw_c = mlp_forward_f16(p_coarse, x).reshape(*shp, -1)
    rgb_c, w_c, depth_c, ins_c, acc_c = O.composite(raw_c, z_coarse, rays_d)
    z_mid = 0.5 * (z_coarse[..., 1:] + z_coarse[..., :-1])
    z_samples = O.sample_pdf(z_mid, w_c[..., 1:-1], n_importance, det=True)
    z_fine, _ = torch.sort(torch.cat([z_coarse, z_samples], -1), -1)
    x, shp = O._net_inputs(rays_o, rays_d, viewdirs, z_fine)
    raw_f = mlp_forward_f16(p_fine, x).reshape(*shp, -1)
    rgb_f, w_f, depth_f, ins_f, acc_f = O.composite(raw_f, z_fine, rays_d)
    return {"rgb_fine": rgb_f, "ins_fine": ins_f, "depth_fine": depth_f, "acc_fine": acc_f, "z_vals_fine": z_fine,
            "rgb_coarse": rgb_c, "ins_coarse": ins_c, "depth_coarse": depth_c, "z_vals_coarse": z_coarse}


def net_inputs_fp32(rays_o, rays_d, z):
    """The network inputs [N * S, 90] as the kernels form them in rays mode and in the fused render (mlp_umma.cu, prologue):
    in fp32, every operation rounded, in the kernel's order -- pts = o + d * z, |d| = sqrt((d0^2 + d1^2) + d2^2), viewdir =
    d / |d| -- then embedded with fp32 sin / cos of x * 2^k (exact scalings).  The kernel's own sin / cos is within 2 ulp of
    these, so a comparison on these inputs is free of the fp32-vs-fp64 input term (up to 2^9 |x| ulp at frequency 2^9)."""
    o, d, z = rays_o.float(), rays_d.float(), z.float()
    pts = o[:, None, :] + d[:, None, :] * z[..., None]
    nrm = torch.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    vd = (d / nrm[:, None])[:, None, :].expand(pts.shape)
    return points_inputs_fp32(pts.reshape(-1, 3), vd.reshape(-1, 3))


def points_inputs_fp32(pts, viewdirs):
    """The network inputs [M, 90] of points mode: the fp32 points and view directions embedded as they are."""
    return torch.cat([O.embed(pts.float(), 10), O.embed(viewdirs.float(), 4)], -1)


def embed_freq_scale(n_freqs):
    """[3 + 6 L]: the factor 2^k each column of O.embed multiplies its input by (1 for the identity columns)."""
    return torch.tensor([1.0] * 3 + [float(2 ** k) for k in range(n_freqs) for _ in range(6)], dtype=torch.float64)


def render_on_depths(net_c, net_f, rays_o, rays_d, z_coarse, z_fine, fp32_inputs=True, keep=None, keep_all_ins=False):
    """Teacher-forced render: the two networks at the caller's coarse [N, S] and fine [N, F] depths (a kernel's own), each pass
    composited in fp64 (O.composite), optionally with the object selection objects_oracle.select_objects(raw, keep) applied
    before the composite.  net_c / net_f: x [M, 90] -> raw [M, C] (mlp_forward_f16 or O.mlp_forward in fp64, closed over the
    weights); either may be None to skip its pass.  fp32_inputs: the networks see net_inputs_fp32 (the kernels' inputs);
    otherwise O._net_inputs in fp64 (O.render's own).  Returns, per pass p in (coarse, fine): rgb_p, depth_p, acc_p, ins_p,
    weights_p, raw_p (unselected), labels_p (per-sample arg-max label, first maximum) and gap_p (per sample, the largest
    instance sigmoid minus the second largest)."""
    from . import objects_oracle as OO
    ro, rd = rays_o.double(), rays_d.double()
    viewdirs = rd / torch.norm(rd, dim=-1, keepdim=True)
    out = {}
    for tag, net, z in (("coarse", net_c, z_coarse), ("fine", net_f, z_fine)):
        if net is None:
            continue
        z = z.double()
        x = net_inputs_fp32(rays_o, rays_d, z) if fp32_inputs else O._net_inputs(ro, rd, viewdirs, z)[0]
        raw = net(x).double().reshape(z.shape[0], z.shape[1], -1)
        sel = raw if keep is None else OO.select_objects(raw, keep)
        rgb, w, depth, ins, acc = O.composite(sel, z, rd, keep_all_ins=keep_all_ins)
        top2 = torch.topk(torch.sigmoid(raw[..., 4:]), 2, dim=-1).values
        out.update({"rgb_" + tag: rgb, "depth_" + tag: depth, "acc_" + tag: acc, "ins_" + tag: ins, "weights_" + tag: w,
                    "raw_" + tag: raw, "labels_" + tag: OO.object_labels(raw), "gap_" + tag: top2[..., 0] - top2[..., 1]})
    return out


def psnr(got, ref):
    """rgb PSNR in dB (peak 1) of got against ref."""
    mse = float(((got.double() - ref.double()) ** 2).mean())
    return 10.0 * torch.log10(torch.tensor(1.0 / max(mse, 1e-300))).item()


def rel_l2(got, ref):
    got, ref = got.double(), ref.double()
    return float(torch.linalg.norm(got - ref) / torch.linalg.norm(ref).clamp_min(1e-300))


def split_rays(rgb_got, rgb_ref, frac=0.0025):
    """(typical, outliers): boolean masks over rays.  The outliers are the at most `frac` of the rays (at least one) with the
    largest rgb error, and only those above 0.05: rays whose importance samples land in another bin (sample_pdf amplifies a
    last-bit difference of the coarse weights, SURVEY.md section 7), which no network precision short of fp64 avoids."""
    err = (rgb_got.double() - rgb_ref.double()).abs().amax(-1)
    k = max(1, int(frac * len(err)))
    worst = torch.zeros_like(err, dtype=torch.bool)
    worst[torch.topk(err, k).indices] = True
    out = worst & (err > 0.05)
    return ~out, out


def label_agreement(ins_got, ins_ref):
    """Fraction of rays whose arg-max instance label agrees."""
    return float((ins_got.argmax(-1) == ins_ref.argmax(-1)).double().mean())
