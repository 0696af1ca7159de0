"""GPU: the training backward against float64 references.

* dmnerf_mlp_backward against a teacher-forced float64 reference built from the very planes the forward saved: every layer
  reads the kernel's saved input plane and is differentiated through the kernel's saved ReLU bits, so the ReLU-flip noise of
  the tensor-core forward drops out and one tight bound holds for both forwards.  Every object-head width the weight
  gradients switch kernels at, batch sizes around the 32-sample stage and the 128-row tile, and the sizes one 1024-ray
  training step runs (65 536 coarse and 196 608 fine samples).
* The gradients are reproducible bit for bit: two calls, two whole training steps, the flag variants.
* dmnerf_composite_backward at ragged shapes (hypothesis, derandomised) against float64 autograd of the oracle.
* End-to-end coarse gradients at the two object-head widths of the replica workloads (ins_num 69 and 93)."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from hypothesis import given, settings, strategies as st, HealthCheck

pytestmark = pytest.mark.gpu

from dmnerf_b200 import synth, _lib
from dmnerf_b200.testing import model_from_weights, scale_err
from oracle import dmnerf_oracle as O

DEV = "cuda"
PLANES = [("h%d" % l, 256) for l in range(8)] + [("rgb_hid", 128), ("ins_hid", 128)]
CHUNK = 16384                      # rows per float64 reference chunk (about 1 GB of autograd state)
TOL_SCALE, TOL_L2 = 2e-4, 1e-4     # the exact-forward bounds of test_mlp_backward_tensor_core_gemms


def _ctx():
    from dmnerf_b200.engine import get_context
    return get_context(torch.device(DEV))


def _net(ins_num, seed):
    w = synth.make_weights(seed, ins_num)
    return model_from_weights(w, DEV).train()


def _params(net):
    from dmnerf_b200.engine import ordered_params
    return ordered_params(net)[0]


def _x_inputs(m, seed):
    gen = torch.Generator().manual_seed(seed)
    pts = torch.rand(m, 3, generator=gen) * 6 - 3
    vd = torch.randn(m, 3, generator=gen)
    vd = vd / vd.norm(dim=-1, keepdim=True)
    return torch.cat([O.embed(pts, 10), O.embed(vd, 4)], -1).to(DEV).contiguous()


def _ray_inputs(n, s, seed):
    wl = synth.workload("dmsr_study")
    sel = np.random.Generator(np.random.PCG64(seed)).choice(wl["rays_o"].shape[0], n, replace=False)
    gen = torch.Generator().manual_seed(seed)
    z = torch.rand(n, s, generator=gen).sort(-1).values * (wl["far"] - wl["near"]) + wl["near"]
    return (torch.from_numpy(wl["rays_o"][sel]).to(DEV).contiguous(), torch.from_numpy(wl["rays_d"][sel]).to(DEV).contiguous(),
            z.to(DEV).contiguous())


def forward_train(net, impl, x=None, rays=None):
    """dmnerf_mlp_forward_train on slot 0 (x [M,90], or rays = (rays_o, rays_d, z [N,S])) -> (acts, out)."""
    ctx = _ctx()
    ins_num = ctx.bind(0, net)
    if x is not None:
        m, s, ro, rd, z = x.shape[0], 1, None, None, None
    else:
        (ro, rd, z), x = rays, None
        m, s = z.numel(), z.shape[1]
    out = torch.empty(m, 5 + ins_num, device=DEV)
    acts = torch.empty(max(m * ctx.lib.dmnerf_act_floats_per_sample(), 1), device=DEV)
    ctx.call("dmnerf_mlp_forward_train", ctx.handle, 0, _lib.ptr(x), _lib.ptr(ro), _lib.ptr(rd), _lib.ptr(z), m, s, _lib.ptr(out),
             _lib.ptr(acts), impl)
    return acts, out


def backward(net, acts, d_out, flags, fill=0.0):
    """dmnerf_mlp_backward through the C ABI into 30 fresh buffers filled with `fill` (bit 1 of flags: they are zero)."""
    ctx = _ctx()
    ctx.bind(0, net)
    m = d_out.shape[0]
    grads = [torch.full(p.shape, fill, device=DEV) for p in _params(net)]
    scratch = torch.empty(max(int(ctx.lib.dmnerf_mlp_backward_scratch_floats(m)), 1), device=DEV)
    ctx.call("dmnerf_mlp_backward", ctx.handle, 0, _lib.ptr(acts), _lib.ptr(d_out), m, _lib.ptrs(grads), _lib.ptr(scratch), flags)
    ctx.sync_check()
    return grads


def planes(acts, m):
    """The saved activations: [M, width] planes h0..h7, rgb_hid, ins_hid, the column-major embedded input and the
    [10][16][M] uint16 ReLU bit planes (bit c of group g = unit 16 g + c)."""
    out, off = {}, 0
    for name, width in PLANES:
        out[name] = acts[off:off + m * width].view(m, width)
        off += m * width
    out["emb"] = acts[off:off + m * 90].view(90, m).t()
    off += m * 90
    out["bits"] = acts[off:off + m * 80].view(torch.int16).view(10, 16, m)
    return out


def relu_mask(bits, plane, width, r0, r1):
    g = bits[plane, :width // 16, r0:r1].to(torch.int32) & 0xFFFF
    b = (g[:, :, None] >> torch.arange(16, device=DEV, dtype=torch.int32)) & 1
    return b.permute(1, 0, 2).reshape(r1 - r0, width)


def reference(net, pl, d_out, m):
    """float64 gradients of sum(out * d_out), teacher-forced on the saved planes (oracle layer order: the skip reads [h, pts],
    the instance branch h.detach()), summed over row chunks in float64.  Also the plane check: the worst scale error of each
    saved plane against the plain float64 forward from the saved embedded input, and whether every bit is plane > 0."""
    names = synth.param_names(net.ins_linear.weight.shape[0] - 1)
    src = dict(net.named_parameters())
    P = {k: src[k].detach().double().requires_grad_(True) for k in names}
    lin = lambda name, t: F.linear(t, P[name + ".weight"], P[name + ".bias"])
    total = [torch.zeros_like(P[k]) for k in names]
    diff = {name: 0.0 for name, _ in PLANES}
    peak = {name: 0.0 for name, _ in PLANES}
    bits_ok = True
    for r0 in range(0, m, CHUNK):
        r1 = min(r0 + CHUNK, m)
        emb = pl["emb"][r0:r1].double()
        pts, dirs = emb[:, :63], emb[:, 63:]
        masks = {}
        for idx, (name, width) in enumerate(PLANES):
            masks[name] = relu_mask(pl["bits"], idx, width, r0, r1)
            bits_ok = bits_ok and torch.equal(masks[name].bool(), pl[name][r0:r1] > 0)

        def relu_tf(z, name):              # value: the kernel's plane; gradient: through the kernel's mask
            mz = masks[name].double() * z
            return pl[name][r0:r1].double() + mz - mz.detach()

        h = pts
        for l in range(8):
            h = relu_tf(lin("mlps.%d" % l, h), "h%d" % l)
            if l == 4:
                h = torch.cat([h, pts], -1)
        rh = relu_tf(lin("rgb_feature_linears.0", torch.cat([lin("rgb_feature_linear", h), dirs], -1)), "rgb_hid")
        ih = relu_tf(lin("ins_feature_linears.0", lin("ins_feature_linear", h.detach())), "ins_hid")
        out = torch.cat([lin("rgb_linear", rh), lin("density_linear", h), lin("ins_linear", ih)], -1)
        loss = (out * d_out[r0:r1].double()).sum()
        for t, g in zip(total, torch.autograd.grad(loss, [P[k] for k in names])):
            t += g
        del h, rh, ih, out, loss
        with torch.no_grad():              # the plain float64 forward of the same inputs
            def seen(name, v):
                diff[name] = max(diff[name], float((pl[name][r0:r1].double() - v).abs().max()))
                peak[name] = max(peak[name], float(v.abs().max()))
            h = pts
            for l in range(8):
                h = torch.relu(lin("mlps.%d" % l, h))
                seen("h%d" % l, h)
                if l == 4:
                    h = torch.cat([h, pts], -1)
            seen("rgb_hid", torch.relu(lin("rgb_feature_linears.0", torch.cat([lin("rgb_feature_linear", h), dirs], -1))))
            seen("ins_hid", torch.relu(lin("ins_feature_linears.0", lin("ins_feature_linear", h))))
    plane_err = {k: diff[k] / max(peak[k], 1e-30) for k in diff}
    return dict(zip(names, total)), plane_err, bits_ok


def grad_errs(got, ref):
    """(scale error, relative L2) of one gradient; a gradient that is exactly zero in float64 must be exactly zero."""
    g = got.double()
    if float(ref.abs().max()) == 0.0:
        return (0.0, 0.0) if float(g.abs().max()) == 0.0 else (math.inf, math.inf)
    d = g - ref
    return float(d.abs().max() / ref.abs().max()), float(d.norm() / ref.norm())


def check_gradients(net, grads, ref, label):
    names = synth.param_names(net.ins_linear.weight.shape[0] - 1)
    errs = {k: grad_errs(g, ref[k]) for k, g in zip(names, grads)}
    ws = max(errs, key=lambda k: errs[k][0])
    wl = max(errs, key=lambda k: errs[k][1])
    print("%s: worst scale err %.2e (%s), worst rel L2 %.2e (%s)" % (label, errs[ws][0], ws, errs[wl][1], wl))
    bad = {k: e for k, e in errs.items() if not (e[0] <= TOL_SCALE and e[1] <= TOL_L2)}
    assert not bad, (label, bad)


def check_planes(plane_err, bits_ok, label):
    worst = max(plane_err.values())
    print("%s: saved planes worst scale err %.2e" % (label, worst))
    assert bits_ok, label
    assert worst <= 1e-4, (label, plane_err)


IMPLS = [pytest.param(_lib.IMPL_SIMT, id="simt"), pytest.param(_lib.IMPL_UMMA, id="umma")]
WIDTHS = [1, 13, 59, 63, 64, 67, 69, 93, 127]


@pytest.mark.parametrize("m", [1, 31, 32, 33, 127, 128, 129, 4097])
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("ins_num", WIDTHS)
def test_backward_matches_teacher_forced_fp64(ins_num, impl, m):
    """All 30 gradients within the exact-forward bounds with either forward.  ins_num 63 / 64 sit on either side of the
    64-logit switch of the ins_linear weight gradient (tensor cores / fp32 CUDA cores); 67 and 127 take the 128x128 fp32 kernel,
    64, 69 and 93 the generic one.  Batch sizes around the 32-sample stage and the 128-row tile."""
    net = _net(ins_num, 40 + ins_num)
    x = _x_inputs(m, 7 * m + ins_num)
    d_out = torch.randn(m, 5 + ins_num, generator=torch.Generator().manual_seed(m + ins_num)).to(DEV)
    acts, _ = forward_train(net, impl, x=x)
    grads = backward(net, acts, d_out, (1 if impl == _lib.IMPL_UMMA else 0) | 2)      # SIMT: masks derived from the planes
    pl = planes(acts, m)
    assert float((pl["emb"] - x).abs().max()) <= 1e-6 * float(x.abs().max())
    ref, plane_err, bits_ok = reference(net, pl, d_out, m)
    label = "ins_num %d %s M %d" % (ins_num, "umma" if impl == _lib.IMPL_UMMA else "simt", m)
    check_planes(plane_err, bits_ok, label)
    check_gradients(net, grads, ref, label)


@pytest.mark.parametrize("ins_num", [13, 93])
@pytest.mark.parametrize("zero", ["instance_columns", "all_but_density"])
def test_backward_with_zero_gradient_columns(ins_num, zero):
    """d_out with every instance column zero, or only the density column non-zero: the gradients that vanish in float64 are
    exactly zero, the rest within the bounds."""
    m = 4097
    net = _net(ins_num, 3)
    d_out = torch.randn(m, 5 + ins_num, generator=torch.Generator().manual_seed(4)).to(DEV)
    if zero == "instance_columns":
        d_out[:, 4:] = 0.0
    else:
        d_out[:, :3] = 0.0
        d_out[:, 4:] = 0.0
    acts, _ = forward_train(net, _lib.IMPL_UMMA, x=_x_inputs(m, 5))
    grads = backward(net, acts, d_out, 3)
    ref, _, _ = reference(net, planes(acts, m), d_out, m)
    vanish = [k for k, g in ref.items() if float(g.abs().max()) == 0.0]
    assert any(k.startswith("ins_linear") for k in vanish) and (zero == "instance_columns" or "rgb_linear.weight" in vanish)
    check_gradients(net, grads, ref, "ins_num %d zero %s" % (ins_num, zero))


@pytest.mark.parametrize("ins_num", [13, 93])
def test_backward_flag_variants_are_bitwise_equal(ins_num):
    """Bit 1 clear with NaN-filled gradient buffers gives the prezeroed result; with the tensor-core forward, masks derived
    from the planes (bit 0 clear) give the result of the masks the forward wrote."""
    m = 4097
    net = _net(ins_num, 8)
    d_out = torch.randn(m, 5 + ins_num, generator=torch.Generator().manual_seed(6)).to(DEV)
    acts, _ = forward_train(net, _lib.IMPL_UMMA, x=_x_inputs(m, 9))
    base = backward(net, acts, d_out, 3)
    unzeroed = backward(net, acts, d_out, 1, fill=float("nan"))
    derived = backward(net, acts, d_out, 2)
    for k, a, b, c in zip(synth.param_names(ins_num), base, unzeroed, derived):
        assert torch.equal(a, b), k
        assert torch.equal(a, c), k


# 1024 rays, the coarse and the fine sample count of one training step; one process after the small cases above, so the
# per-device partial-product buffer of the weight-gradient GEMMs is first grown and then reused at other sizes.
@pytest.mark.parametrize("ins_num,s", [(13, 64), (13, 192), (93, 64), (93, 192)])
def test_backward_at_training_step_size(ins_num, s):
    """Rays mode, tensor-core forward, 1024 rays x S: the 30 gradients within the bounds and bitwise equal over two calls on
    the same activations; the saved planes right at this size."""
    n = 1024
    m = n * s
    net = _net(ins_num, 60 + ins_num)
    acts, _ = forward_train(net, _lib.IMPL_UMMA, rays=_ray_inputs(n, s, 11))
    d_out = torch.randn(m, 5 + ins_num, generator=torch.Generator().manual_seed(s + ins_num)).to(DEV)
    first = backward(net, acts, d_out, 3)
    second = backward(net, acts, d_out, 3)
    for k, a, b in zip(synth.param_names(ins_num), first, second):
        assert torch.equal(a, b), k
    del second
    ref, plane_err, bits_ok = reference(net, planes(acts, m), d_out, m)
    label = "ins_num %d umma rays 1024 x %d (M %d)" % (ins_num, s, m)
    check_planes(plane_err, bits_ok, label)
    check_gradients(net, first, ref, label)
    del acts, d_out, first, ref
    torch.cuda.empty_cache()


def _step_draws(n, s, n_imp, seed):
    gen = torch.Generator().manual_seed(seed)
    return torch.rand(n, s, generator=gen).to(DEV), torch.rand(n, n_imp, generator=gen).to(DEV)


@pytest.mark.parametrize("ins_num", [13, 93])
def test_training_step_gradients_are_reproducible(ins_num):
    """render_rays_grad (forward + backward of both networks), 1024 rays, perturb = 1 with given draws, twice: all 60
    gradients bitwise equal."""
    from dmnerf_b200.backward import render_rays_grad
    wl = synth.workload("dmsr_study")
    n = 1024
    nc, nf = _net(ins_num, 70), _net(ins_num, 71)
    ro, rd, _ = _ray_inputs(n, 64, 12)
    zc = torch.linspace(wl["near"], wl["far"], 64, device=DEV)
    t_rand, u = _step_draws(n, 64, 128, 13)
    gen = torch.Generator().manual_seed(14)
    G = {k: torch.randn(shape, generator=gen).to(DEV) for k, shape in (("rgb_coarse", (n, 3)), ("rgb_fine", (n, 3)), ("depth_fine", (n,)),
                                                                     ("acc_coarse", (n,)), ("ins_coarse", (n, ins_num)), ("ins_fine", (n, ins_num)))}
    runs = []
    for _ in range(2):
        for p in list(nc.parameters()) + list(nf.parameters()):
            p.grad = None
        out = render_rays_grad(ro, rd, nc, nf, zc, perturb=1.0, N_importance=128, t_rand=t_rand, u=u)
        sum((out[k] * g).sum() for k, g in G.items()).backward()
        runs.append((out["rgb_fine"].detach().clone(), [p.grad.clone() for p in _params(nc) + _params(nf)]))
    assert torch.equal(runs[0][0], runs[1][0])
    names = ["coarse." + k for k in synth.param_names(ins_num)] + ["fine." + k for k in synth.param_names(ins_num)]
    for k, a, b in zip(names, runs[0][1], runs[1][1]):
        assert torch.equal(a, b), k


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("ins_num", [69, 93])
def test_coarse_step_gradients_at_wide_object_heads(ins_num, impl):
    """render_rays_grad at the object-head widths of the two replica configs, 64 rays, perturb = 1 with given draws, loss on the
    coarse outputs only (no sample_pdf on its path): the coarse network's gradients against float64 autograd of the coarse pass
    of the oracle's render (render.py:40-63) with the coarse-network bounds of test_training_step_matches_reference_gradients;
    the fine network's exactly zero.  The reference forms the stratified depths and the embedded inputs in fp32 like the
    original (a float64 sample position differs from the fp32 one by ~1e-6, which sin(2^9 x) turns into ~5e-4 of a feature) and
    everything after them in float64."""
    from dmnerf_b200.backward import render_rays_grad
    wl = synth.workload("dmsr_study")
    n = 64
    nc, nf = _net(ins_num, 80), _net(ins_num, 81)
    ro, rd, _ = _ray_inputs(n, 64, 15)
    zc = torch.linspace(wl["near"], wl["far"], 64, device=DEV)
    t_rand, u = _step_draws(n, 64, 128, 16)
    gen = torch.Generator().manual_seed(17)
    G = {k: torch.randn(shape, generator=gen, dtype=torch.float64) for k, shape in
         (("rgb_coarse", (n, 3)), ("depth_coarse", (n,)), ("acc_coarse", (n,)), ("ins_coarse", (n, ins_num)), ("weights_coarse", (n, 64)))}
    out = render_rays_grad(ro, rd, nc, nf, zc, perturb=1.0, N_importance=128, t_rand=t_rand, u=u, impl=impl)
    sum((out[k] * g.float().to(DEV)).sum() for k, g in G.items()).backward()
    names = synth.param_names(ins_num)
    pc = {k: v.detach().cpu().double().requires_grad_(True) for k, v in nc.named_parameters()}
    ro_c, rd_c = ro.cpu(), rd.cpu()
    z = O.stratify(zc.cpu().expand(n, 64), t_rand.cpu())                                    # render.py:40-47, fp32
    np.testing.assert_allclose(out["z_vals_coarse"].cpu().numpy(), z.numpy(), rtol=0, atol=2e-6)
    z = out["z_vals_coarse"].cpu()
    x, shp = O._net_inputs(ro_c, rd_c, rd_c / torch.norm(rd_c, dim=-1, keepdim=True), z)     # render.py:37,49-58, fp32
    raw = O.mlp_forward(pc, x.double()).reshape(*shp, -1)
    rgb, w, depth, ins, acc = O.composite(raw, z.double(), rd_c.double())                    # render.py:63
    ref = {"rgb_coarse": rgb, "depth_coarse": depth, "acc_coarse": acc, "ins_coarse": ins, "weights_coarse": w}
    sum((ref[k] * g).sum() for k, g in G.items()).backward()
    tol = 1e-3 if impl == _lib.IMPL_SIMT else 1e-2
    got = dict(nc.named_parameters())
    worst = {k: scale_err(got[k].grad.cpu().numpy(), pc[k].grad.numpy()) for k in names}
    print("coarse step ins_num %d %s: worst scale err %.2e (%s)" % (ins_num, "umma" if impl == _lib.IMPL_UMMA else "simt",
                                                                   max(worst.values()), max(worst, key=worst.get)))
    assert all(v <= tol for v in worst.values()), worst
    for k, p in nf.named_parameters():
        assert p.grad is not None and int(torch.count_nonzero(p.grad)) == 0, k


# ------------------------------------------------------------------------------------------------ composite backward
GRAD_KEYS = ("rgb", "depth", "acc", "ins", "weights")


def _composite_case(n, s, k, keep, seed, present, accumulate):
    """One dmnerf_composite_backward call through the C ABI (as backward.py makes it) against float64 autograd of the oracle's
    composite on the same fp32 inputs, with weights and acc_map as differentiable outputs."""
    gen = torch.Generator().manual_seed(seed)
    c = 4 + k
    raw = torch.randn(n, s, c, generator=gen) * 2
    sig = torch.randn(n, s, generator=gen) * 3 - 1                       # plenty of negative densities (clamped)
    sig[torch.rand(n, s, generator=gen) < 0.05] = 0.0                    # and exact zeros
    hit = torch.rand(n, generator=gen) < 0.5                             # rays whose alpha saturates to 1 mid-ray
    at = torch.randint(0, s, (n,), generator=gen)
    sig[hit, at[hit]] = 1e4
    raw[..., 3] = sig
    z = torch.rand(n, s, generator=gen).sort(-1).values * 9 + 1
    rd = torch.randn(n, 3, generator=gen) * 1.5
    n_ins = k if keep else k - 1
    shapes = {"rgb": (n, 3), "depth": (n,), "acc": (n,), "ins": (n, n_ins), "weights": (n, s)}
    g = {key: (torch.randn(shapes[key], generator=gen) if key in present else None) for key in GRAD_KEYS}
    pre = torch.randn(n, s, c, generator=gen) if accumulate else torch.zeros(n, s, c)
    cu = lambda t: None if t is None else t.to(DEV).contiguous()
    raw_d, z_d, rd_d = cu(raw), cu(z), cu(rd)
    gd = {key: cu(v) for key, v in g.items()}
    # float64 reference (on the device)
    r64 = raw_d.double().requires_grad_(True)
    if s == 1:
        # the oracle builds its 1e10 tail distance from dists[..., :1], which is empty for one sample; a second sample 1e10
        # behind the first with zero density (weight 0) gives the lone sample the tail distance and adds nothing
        pad = torch.zeros(n, 1, c, device=DEV, dtype=torch.float64)
        rgb, w, depth, ins, acc = O.composite(torch.cat([r64, pad], 1), torch.cat([z_d.double(), z_d.double() + 1e10], 1),
                                              rd_d.double(), keep_all_ins=keep)
        w = w[:, :1]
    else:
        rgb, w, depth, ins, acc = O.composite(r64, z_d.double(), rd_d.double(), keep_all_ins=keep)
    outs = {"rgb": rgb, "depth": depth, "acc": acc, "ins": ins, "weights": w}
    loss = r64.sum() * 0.0
    for key in GRAD_KEYS:
        if gd[key] is not None:
            loss = loss + (outs[key] * gd[key].double()).sum()
    ref = torch.autograd.grad(loss, r64)[0]
    # scale the preload like each channel group's gradient, so that a preload does not hide its errors
    for sl in (slice(0, 3), slice(3, 4), slice(4, None)):
        pre[..., sl] *= max(float(ref[..., sl].abs().max()), 1e-6)
    d_raw = cu(pre.float())
    pre_d = d_raw.clone()
    _ctx().call("dmnerf_composite_backward", _lib.ptr(raw_d), _lib.ptr(z_d), _lib.ptr(rd_d), n, s, c, int(keep), _lib.ptr(gd["rgb"]),
                _lib.ptr(gd["depth"]), _lib.ptr(gd["acc"]), _lib.ptr(gd["ins"]), _lib.ptr(gd["weights"]), _lib.ptr(d_raw), int(accumulate))
    _ctx().sync_check()
    got = d_raw.double() - pre_d.double() if accumulate else d_raw.double()
    for sl in (slice(0, 3), slice(3, 4), slice(4, None)):
        r = ref[..., sl]
        peak = float(r.abs().max())
        err = float((d_raw.double()[..., sl] - pre_d.double()[..., sl] - r).abs().max())
        if peak == 0.0:
            assert torch.equal(d_raw[..., sl], pre_d[..., sl]), sl          # nothing flows in: the preload (or 0) untouched
        else:
            assert err <= 1e-4 * peak, (sl, err / peak)
    off = raw_d[..., 3] <= 0.0
    assert torch.equal(d_raw[..., 3][off], pre_d[..., 3][off])               # relu: exactly no density gradient
    if not keep:
        assert torch.equal(d_raw[..., -1], pre_d[..., -1])                  # the dropped last channel (render.py:26)
    assert torch.isfinite(got).all()


@pytest.mark.parametrize("s", [1, 2, 31, 32, 33, 64, 192, 2048])
def test_composite_backward_fixed_sample_counts(s):
    """Sample counts around the 32-lane chunks of the reverse scan, the training counts, and 2048 (160 KB of shared memory);
    both topologies, every upstream gradient, with and without accumulate."""
    for i, (keep, accumulate) in enumerate(((False, False), (True, True), (False, True), (True, False))):
        _composite_case(n=9 + i, s=s, k=(13, 94, 1, 128)[i], keep=keep, seed=100 * s + i, present=set(GRAD_KEYS), accumulate=accumulate)


@settings(max_examples=25, deadline=None, suppress_health_check=list(HealthCheck), derandomize=True)
@given(n=st.integers(1, 70), s=st.integers(1, 300), k=st.integers(1, 128), keep=st.booleans(), seed=st.integers(0, 2 ** 20),
       present=st.sets(st.sampled_from(GRAD_KEYS)), accumulate=st.booleans())
def test_composite_backward_fuzz(n, s, k, keep, seed, present, accumulate):
    """Ragged rays / samples / instance channels, any subset of the five upstream gradients passed as NULL."""
    _composite_case(n, s, k, keep, seed, present, accumulate)
