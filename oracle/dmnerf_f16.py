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
