"""GPU: the training path (BASELINE config 4) -- native forward with saved activations + native backward, compared with
torch autograd on the oracle (CPU) and with the reference's own gradients stored in tests/golden/render_study.npz."""
import os
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from dmnerf_b200 import synth, _lib
from dmnerf_b200.testing import model_from_weights, scale_err, rel_l2
from oracle import dmnerf_oracle as O

DEV = "cuda"


def load(golden_dir, name):
    return dict(np.load(os.path.join(golden_dir, name)))


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def test_composite_backward_matches_autograd(golden_dir):
    from dmnerf_b200.render import render_train
    g = load(golden_dir, "composite.npz")
    gen = torch.Generator().manual_seed(3)
    raw = torch.from_numpy(g["raw"]).clone().requires_grad_(True)
    z, rd = torch.from_numpy(g["z"]), torch.from_numpy(g["rays_d"])
    G = [torch.randn(s, generator=gen) for s in ((24, 3), (24,), (24, 13))]
    rgb, w, depth, ins, acc = O.composite(raw, z, rd)
    ((rgb * G[0]).sum() + (depth * G[1]).sum() + (ins * G[2]).sum()).backward()
    raw_c = cu(g["raw"]).requires_grad_(True)
    rgb2, w2, depth2, ins2 = render_train(raw_c, cu(g["z"]), cu(g["rays_d"]))
    ((rgb2 * G[0].to(DEV)).sum() + (depth2 * G[1].to(DEV)).sum() + (ins2 * G[2].to(DEV)).sum()).backward()
    got, ref = raw_c.grad.cpu().numpy(), raw.grad.numpy()
    for sl in (slice(0, 3), slice(3, 4), slice(4, None)):
        assert scale_err(got[..., sl], ref[..., sl]) <= 1e-4, sl
    assert float(np.abs(got[..., -1]).max()) == 0.0          # dropped last class gets no gradient (render.py:26)
    # manipulator_render variant: weights not detached, all channels kept
    raw = torch.from_numpy(g["raw"]).clone().requires_grad_(True)
    out = O.composite(raw, z, rd, keep_all_ins=True)
    Gi = torch.randn((24, 14), generator=gen)
    ((out[0] * G[0]).sum() + (out[3] * Gi).sum()).backward()
    raw_c = cu(g["raw"]).requires_grad_(True)
    o2 = render_train(raw_c, cu(g["z"]), cu(g["rays_d"]), keep_all_ins=True)
    ((o2[0] * G[0].to(DEV)).sum() + (o2[3] * Gi.to(DEV)).sum()).backward()
    assert scale_err(raw_c.grad.cpu().numpy(), raw.grad.numpy()) <= 1e-4


IMPLS = [pytest.param(_lib.IMPL_SIMT, id="simt"), pytest.param(_lib.IMPL_UMMA, id="umma")]


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("ins_num", [13, 59])
def test_mlp_backward_matches_autograd(golden_dir, ins_num, impl):
    g = load(golden_dir, "mlp_ins%d.npz" % ins_num)
    w = synth.make_weights(int(g["seed"]), ins_num)
    p = O.to_torch(w)
    for v in p.values():
        v.requires_grad_(True)
    x = torch.from_numpy(g["x"])
    G = torch.randn(g["y"].shape, generator=torch.Generator().manual_seed(5))
    (O.mlp_forward(p, x) * G).sum().backward()
    net = model_from_weights(w, DEV).train()
    y = net(cu(g["x"]), impl=impl)
    assert y.requires_grad
    np.testing.assert_allclose(y.detach().cpu().numpy(), g["y"], rtol=1e-4, atol=5e-5)
    (y * G.to(DEV)).sum().backward()
    # exact-fp32 forward: gradients agree to fp32 noise.  Tensor-core forward: its ~1e-5 activation noise flips the ReLU mask
    # of the few units whose pre-activation is within 1e-5 of zero; each flip moves individual gradient entries by O(1e-3)
    # of the tensor's scale (injecting 1e-5 relative noise into the oracle's pre-activations reproduces relL2 5e-4...3e-3),
    # so the bound is relative L2 5e-3 (max-norm 5e-2: a single flip dominates single entries in a 130-row batch) there; DMNERF_TRAIN_IMPL=simt selects the exact-fp32 forward.
    tol_max, tol_l2 = (2e-4, 1e-4) if impl == _lib.IMPL_SIMT else (5e-2, 5e-3)
    for k, prm in net.named_parameters():
        ref = p[k].grad.numpy()
        assert prm.grad is not None, k
        got = prm.grad.cpu().numpy()
        assert scale_err(got, ref) <= tol_max and rel_l2(got, ref) <= tol_l2, (k, scale_err(got, ref), rel_l2(got, ref))


@pytest.mark.parametrize("impl", IMPLS)
def test_training_step_matches_reference_gradients(golden_dir, impl):
    """C4: 16 rays, perturb=1 with the reference's own uniform draws, loss of oracle.train_loss; gradients of all 60
    parameter tensors against the reference's (strided slices + norms stored in the fixture)."""
    from dmnerf_b200.backward import render_rays_grad
    g = load(golden_dir, "render_study.npz")
    ins_num = int(g["ins_num"])
    nc = model_from_weights(synth.make_weights(int(g["seed_coarse"]), ins_num), DEV).train()
    nf = model_from_weights(synth.make_weights(int(g["seed_fine"]), ins_num), DEV).train()
    ro, rd = cu(g["rays_o"]), cu(g["rays_d"])
    zc = cu(g["det_z_vals_coarse"][0])
    out = render_rays_grad(ro, rd, nc, nf, zc, perturb=1.0, N_importance=128, t_rand=cu(g["t_rand"]), u=cu(g["u"]), impl=impl)
    np.testing.assert_allclose(out["z_vals_coarse"].cpu().numpy(), g["trn_z_vals_coarse"], rtol=0, atol=2e-6)
    np.testing.assert_allclose(out["rgb_coarse"].detach().cpu().numpy(), g["trn_rgb_coarse"], rtol=1e-4, atol=1e-5)
    loss = O.train_loss(out, cu(g["target"]))
    assert abs(float(loss) - float(g["loss"])) <= 2e-3 * abs(float(g["loss"]))
    loss.backward()
    worst = {}
    for nm, net in (("coarse", nc), ("fine", nf)):
        for k, prm in net.named_parameters():
            ref = g["grad_%s_%s" % (nm, k)]
            got = prm.grad.cpu().numpy()
            if k.endswith("weight"):
                n_ref = float(g["gnorm_%s_%s" % (nm, k)])
                assert abs(float(np.linalg.norm(got)) - n_ref) <= 2e-2 * n_ref + 1e-7, (nm, k)
                got = got[::8, ::8]
            tol = (1e-3 if impl == _lib.IMPL_SIMT else 1e-2) if nm == "coarse" else 3e-2   # fine: ill-conditioned sample_pdf
            worst[(nm, k)] = scale_err(got, ref) if np.abs(ref).max() > 0 else float(np.abs(got).max())
            assert worst[(nm, k)] <= tol, (nm, k, worst[(nm, k)])
    # detach topology: the instance loss never reaches the trunk via ins_feature_linear's input (dm_nerf.py:95)
    assert float(nc.mlps[0].weight.grad.abs().max()) > 0


def test_dropin_training_loop_runs_and_rebinds_updated_weights():
    """train_*.py usage: dm_nerf() under autograd with args.perturb=1, Adam over both networks, two iterations."""
    from dmnerf_b200.render import dm_nerf
    from dmnerf_b200.embedder import get_embedder
    from dmnerf_b200.helpers import z_val_sample
    from dmnerf_b200.testing import make_models
    wl = synth.workload("dmsr_study")
    nc, nf, _, _ = make_models(7, 8, 13, DEV)
    nc.train(); nf.train()
    opt = torch.optim.Adam(list(nc.parameters()) + list(nf.parameters()), lr=5e-4)
    sel = np.random.Generator(np.random.PCG64(0)).choice(307200, 256, replace=False)
    rays = torch.stack([cu(wl["rays_o"][sel]), cu(wl["rays_d"][sel])], 0)
    args = types.SimpleNamespace(perturb=1.0, N_importance=128, is_train=True, N_ins=None)
    pe, ve = get_embedder(10)[0], get_embedder(4)[0]
    zc = z_val_sample(256, wl["near"], wl["far"], 64, device=DEV)
    target = torch.rand(256, 3, device=DEV)
    losses = []
    torch.manual_seed(3)
    for _ in range(3):
        out = dm_nerf(rays, pe, ve, nc, nf, zc, args)
        assert set(("rgb_fine", "ins_fine", "raw_fine", "raw_coarse", "depth_fine")) <= set(out)
        loss = ((out["rgb_fine"] - target) ** 2).mean() + ((out["rgb_coarse"] - target) ** 2).mean() \
            + 0.1 * out["ins_fine"].mean() + 1e-3 * out["raw_fine"][..., 4:].pow(2).mean()
        opt.zero_grad()
        loss.backward()
        assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in nc.parameters())
        opt.step()
        losses.append(float(loss))
    assert losses[-1] < losses[0]            # Adam on a fixed batch must make progress => the re-bound weights are live


@pytest.mark.parametrize("m", [300, 128 * 5])
def test_tensor_core_training_forward_saves_the_reference_activations(m):
    """dmnerf_mlp_forward_train(impl=UMMA, rays mode): the planes kept for the backward -- the embedded inputs produced by the
    kernel's own branch-free sin/cos (dm_nerf.py:37-38), H0..H7 (dm_nerf.py:84-87) and the two hidden head activations
    (dm_nerf.py:93,99) -- against the oracle on the same rays; a ragged last tile included."""
    from dmnerf_b200.engine import get_context
    wl = synth.workload("dmsr_study")
    w = synth.make_weights(11, 13)
    net = model_from_weights(w, DEV)
    ctx = get_context(torch.device(DEV))
    lib = ctx.lib
    S = 4
    n = (m + S - 1) // S
    m = n * S
    sel = np.linspace(0, 307199, n).astype(np.int64)
    ro, rd = cu(wl["rays_o"][sel]), cu(wl["rays_d"][sel])
    z = (torch.rand(n, S, generator=torch.Generator().manual_seed(5)).sort(-1).values * 11 + 4).to(DEV).contiguous()
    assert ctx.bind(0, net) == 13
    apf = lib.dmnerf_act_floats_per_sample()
    raw = torch.empty(m, 18, device=DEV)
    acts = torch.zeros(m * apf, device=DEV)
    _lib.check(lib.dmnerf_mlp_forward_train(ctx.handle, 0, None, _lib.ptr(ro), _lib.ptr(rd), _lib.ptr(z), m, S, _lib.ptr(raw),
                                            _lib.ptr(acts), _lib.IMPL_UMMA, ctx.stream()), "dmnerf_mlp_forward_train")
    ctx.sync_check()
    acts = acts.cpu().numpy()
    off = 0
    planes = {}
    for name, width in [("h%d" % l, 256) for l in range(8)] + [("rgb_feat", 256), ("ins_feat", 256), ("rgb_hid", 128),
                                                              ("ins_hid", 128), ("emb", 90)]:
        block = acts[off:off + m * width]
        planes[name] = block.reshape(width, m).T if name == "emb" else block.reshape(m, width)      # emb is stored column-major
        off += m * width
    # oracle on the CPU
    p = O.to_torch(w)
    pts = (torch.from_numpy(wl["rays_o"][sel])[:, None, :] + torch.from_numpy(wl["rays_d"][sel])[:, None, :] * z.cpu()[..., None])
    vd = torch.from_numpy(wl["rays_d"][sel])
    vd = (vd / vd.norm(dim=-1, keepdim=True))[:, None, :].expand(n, S, 3)
    x = torch.cat([O.embed(pts, 10), O.embed(vd, 4)], -1).reshape(m, 90)
    emb = planes["emb"]
    # |sin|,|cos| <= 1: the periodic terms must agree to ~2 ulp of 1 (arguments reach 2^9 * |x| ~ 5e3)
    assert np.abs(emb[:, 3:63] - x.numpy()[:, 3:63]).max() <= 1e-6
    assert np.abs(emb[:, 66:] - x.numpy()[:, 66:]).max() <= 1e-6
    np.testing.assert_allclose(emb[:, :3], x.numpy()[:, :3], rtol=0, atol=1e-6)
    h = x[:, :63]
    for i in range(8):
        h = torch.relu(torch.nn.functional.linear(h, p["mlps.%d.weight" % i], p["mlps.%d.bias" % i]))
        assert scale_err(planes["h%d" % i], h.numpy()) <= 1e-4, i
        if i == 4:
            h = torch.cat([h, x[:, :63]], -1)
    rf = torch.nn.functional.linear(h, p["rgb_feature_linear.weight"], p["rgb_feature_linear.bias"])
    rh = torch.relu(torch.nn.functional.linear(torch.cat([rf, x[:, 63:]], -1), p["rgb_feature_linears.0.weight"],
                                               p["rgb_feature_linears.0.bias"]))
    inf = torch.nn.functional.linear(h, p["ins_feature_linear.weight"], p["ins_feature_linear.bias"])
    ih = torch.relu(torch.nn.functional.linear(inf, p["ins_feature_linears.0.weight"], p["ins_feature_linears.0.bias"]))
    assert scale_err(planes["rgb_hid"], rh.numpy()) <= 1e-4
    assert scale_err(planes["ins_hid"], ih.numpy()) <= 1e-4
    out = O.mlp_forward(p, x).numpy()
    assert scale_err(raw.cpu().numpy(), out) <= 1e-4
    # ReLU masks, 1 bit per unit (what the fused gradient chain reads): [10 planes][16 groups][m] uint16, rows fastest, after
    # the embedded inputs; bit c of group g = unit 16 g + c
    bits = acts[off:off + 10 * m * 8].view(np.uint16).reshape(10, 16, m)
    for pl, name in enumerate(["h%d" % l for l in range(8)] + ["rgb_hid", "ins_hid"]):
        width = planes[name].shape[1]
        grp = bits[pl][:width // 16].astype(np.uint32)                                        # [groups, m]
        unpacked = ((grp[:, :, None] >> np.arange(16, dtype=np.uint32)) & 1).transpose(1, 0, 2).reshape(m, width)
        assert np.array_equal(unpacked.astype(bool), planes[name] > 0), name


@pytest.mark.parametrize("ins_num", [13, 59, 127])
def test_mlp_backward_tensor_core_gemms(ins_num):
    """Batches of >= 512 samples run the backward on the tensor cores: the split-bf16 wgmma dX and dW GEMMs (gemm_umma.cu) layer
    by layer; with the exact-fp32 forward the 30 parameter gradients must still agree with torch autograd on the oracle to fp32
    noise.  1333 samples: ten full 128-row tiles + a ragged one, 32-sample stages with a ragged tail; ins_num = 127 is the widest
    object head the library accepts (128 instance logits)."""
    m = 1333
    w = synth.make_weights(21, ins_num)
    p = O.to_torch(w)
    for v in p.values():
        v.requires_grad_(True)
    gen = torch.Generator().manual_seed(9)
    pts = torch.rand(m, 3, generator=gen) * 6 - 3
    vd = torch.randn(m, 3, generator=gen)
    vd = vd / vd.norm(dim=-1, keepdim=True)
    x = torch.cat([O.embed(pts, 10), O.embed(vd, 4)], -1)
    G = torch.randn(m, 4 + ins_num + 1, generator=gen)
    (O.mlp_forward(p, x) * G).sum().backward()
    net = model_from_weights(w, DEV).train()
    y = net(x.to(DEV), impl=_lib.IMPL_SIMT)
    (y * G.to(DEV)).sum().backward()
    from dmnerf_b200.engine import get_context
    get_context(torch.device(DEV)).sync_check()
    for k, prm in net.named_parameters():
        ref = p[k].grad.numpy()
        got = prm.grad.cpu().numpy()
        assert scale_err(got, ref) <= 2e-4 and rel_l2(got, ref) <= 1e-4, (k, scale_err(got, ref), rel_l2(got, ref))


@pytest.mark.parametrize("tag", ["a", "b"])
def test_emptiness_penalizer_matches_reference(golden_dir, tag):
    """networks/penalizer.py (train_dmsr.py:53-60): loss and its gradient w.r.t. raw against the reference's own values
    (tests/golden/penalizer.npz, generated by oracle/make_golden_penalizer.py); rays whose depth lies before / behind every
    sample are included."""
    from dmnerf_b200.penalizer import ins_penalizer
    g = load(golden_dir, "penalizer.npz")
    args = types.SimpleNamespace(tolerance=float(g["tolerance"]), deta_w=float(g["deta_w"]))
    raw = cu(g["raw_" + tag]).requires_grad_(True)
    before = _lib.launch_count()
    loss = ins_penalizer(raw, cu(g["z_" + tag]), cu(g["depth_" + tag]), cu(g["rays_d_" + tag]), args)
    assert loss.shape == (1,)
    assert _lib.launch_count() == before + 1          # populations, sums and finalisation in one pass
    ref = float(g["loss_" + tag][0])
    assert abs(float(loss.detach()) - ref) <= 1e-5 * abs(ref)
    (loss.sum() * 3.0).backward()
    got, want = raw.grad.cpu().numpy(), 3.0 * g["grad_" + tag]
    assert np.abs(got[..., :4]).max() == 0.0
    assert scale_err(got, want) <= 1e-5 and rel_l2(got, want) <= 1e-5, (scale_err(got, want), rel_l2(got, want))
    # empty batch
    z0 = torch.zeros(0, 64, device=DEV)
    l0 = ins_penalizer(torch.zeros(0, 64, 18, device=DEV), z0, torch.zeros(0, device=DEV), torch.zeros(0, 3, device=DEV), args)
    assert float(l0) == 0.0


@pytest.mark.parametrize("tag", ["a", "b", "c"])
def test_hungarian_instance_loss_matches_reference(golden_dir, tag):
    """networks/evaluator.py:19-74 on the native kernels: cost matrices, assignment, loss parts and d loss / d pred against the
    values the unmodified reference produced (tests/golden/evaluator.npz, oracle/make_golden_evaluator.py)."""
    from dmnerf_b200.evaluator import ins_criterion, hungarian
    g = load(golden_dir, "evaluator.npz")
    k = int(g["k_" + tag])
    pred = cu(g["pred_" + tag]).requires_grad_(True)
    lab = cu(g["labels_" + tag])
    before = _lib.launch_count()
    parts = ins_criterion(pred, lab, k)
    parts[0].sum().backward()
    assert _lib.launch_count() - before >= 2
    got = np.array([float(x.detach().float().sum()) for x in parts])
    np.testing.assert_allclose(got, g["loss_" + tag], rtol=1e-5, atol=1e-7)
    gref = g["grad_" + tag]
    assert scale_err(pred.grad.cpu().numpy(), gref) <= 1e-5
    np.testing.assert_allclose(pred.grad.cpu().numpy(), gref, rtol=2e-4, atol=1e-9)
    valid = torch.unique(lab)
    gt = torch.zeros(lab.shape[0], k, device=DEV)
    gt[:, :len(valid)] = torch.nn.functional.one_hot(lab.long())[..., valid.long()].float()
    ce, siou, rows, cols = hungarian(pred.detach(), gt, len(valid), k)
    np.testing.assert_allclose(ce.cpu().numpy(), g["cost_ce_" + tag], rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(siou.cpu().numpy(), g["cost_siou_" + tag], rtol=1e-5, atol=1e-6)
    assert list(cols[:len(valid)]) == list(g["order_col_" + tag][:len(valid)])
    assert sorted(cols) == list(range(k))


def _device_assign(cost, n_valid):
    """hungarian_assign_kernel on an arbitrary score matrix (as cost_ce, with cost_siou = 0) through the C ABI."""
    from dmnerf_b200.engine import get_context
    k = cost.shape[0]
    ctx = get_context(torch.device(DEV))
    ce = cu(cost.astype(np.float32))
    si = torch.zeros_like(ce)
    col_sum = torch.ones(k, device=DEV)
    nv = torch.tensor([n_valid], device=DEV, dtype=torch.int32)
    row_of_col = torch.full((k,), -7, device=DEV, dtype=torch.int32)
    losses = torch.empty(3, device=DEV)
    _lib.check(ctx.lib.dmnerf_hungarian_assign(_lib.ptr(ce), _lib.ptr(si), _lib.ptr(col_sum), nv.data_ptr(), 10, k,
                                               row_of_col.data_ptr(), _lib.ptr(losses), ctx.stream()), "dmnerf_hungarian_assign")
    return row_of_col.cpu().numpy(), losses.cpu().numpy()


def test_device_assignment_is_scipys_assignment_including_ties():
    """The one-warp shortest-augmenting-path solver against scipy.optimize.linear_sum_assignment (evaluator.py:45) on random,
    small-integer (tie-heavy), constant and duplicate-column score matrices of every shape class: the SAME columns, not just the
    same total, because the matched channel decides where the gradient goes."""
    from scipy.optimize import linear_sum_assignment
    from oracle import lsap
    rng = np.random.default_rng(3)
    cases = 0
    for trial in range(160):
        k = int(rng.integers(1, 129)) if trial % 5 else int(rng.choice([1, 2, 32, 33, 94, 127, 128]))
        v = int(rng.integers(1, k + 1)) if trial % 3 else k
        kind = trial % 4
        if kind == 0:
            c = rng.random((k, k))
        elif kind == 1:
            c = rng.integers(0, 3, (k, k)).astype(np.float64)
        elif kind == 2:
            c = np.full((k, k), float(rng.integers(0, 2)))
        else:
            c = rng.random((k, k))
            c[:, rng.integers(0, k, max(1, k // 2))] = c[:, [0]]
        c = c.astype(np.float32)
        rows, cols = linear_sum_assignment(c[:v])
        got, losses = _device_assign(c, v)
        want = np.full(k, -1)
        want[cols] = rows
        assert np.array_equal(got, want), (trial, k, v, kind)
        if k <= 40:        # and the oracle's restatement of scipy's algorithm (oracle/lsap.py, order-free arg-min form)
            assert np.array_equal(lsap.lsap_lane_parallel(c[:v])[1], cols), (trial, k, v, kind)
        np.testing.assert_allclose(losses[0], c[rows, cols].mean(), rtol=1e-6, atol=1e-7)
        assert losses[2] == 0.0
        np.testing.assert_allclose(losses[1], (k - v) / (10.0 * (k - v)) if k > v else 0.0, rtol=1e-6)
        cases += 1
    assert cases == 160
    # non-finite scores: no assignment, NaN losses (scipy raises "matrix contains invalid numeric entries")
    bad = np.ones((4, 4), np.float32); bad[1, :] = np.nan
    got, losses = _device_assign(bad, 4)
    assert (got == -1).all() and np.isnan(losses).all()


def test_instance_loss_device_and_host_assignment_agree_and_nothing_synchronises(monkeypatch):
    """ins_criterion with the assignment on the device (default) against DMNERF_INS_ASSIGN=host (scipy, the reference's
    arrangement): same loss parts, same gradient; labels need not be dense or below ins_num; and the device path raises under
    torch's synchronisation detector neither in forward nor in backward (the host path does: its .cpu() hop)."""
    from dmnerf_b200.evaluator import ins_criterion, ins_assignment
    gen = torch.Generator().manual_seed(21)
    for n, k, label_values in ((1024, 13, [0, 3, 4, 9]), (777, 94, list(range(0, 94, 3))), (64, 5, [7, 200, 65535]), (300, 7, list(range(7)))):
        lv = torch.tensor(label_values)
        lab = lv[torch.randint(0, len(lv), (n,), generator=gen)]
        logits = torch.randn(n, k, generator=gen) * 2
        pred = torch.sigmoid(logits)
        out = {}
        for mode in ("device", "host"):
            monkeypatch.setenv("DMNERF_INS_ASSIGN", mode)
            p = cu(pred.numpy()).requires_grad_(True)
            parts = ins_criterion(p, cu(lab.numpy()), k)
            parts[0].sum().backward()
            out[mode] = ([float(x.detach().float().sum()) for x in parts], p.grad.clone())
        np.testing.assert_allclose(out["device"][0], out["host"][0], rtol=2e-6, atol=1e-7)
        assert float((out["device"][1] - out["host"][1]).abs().max()) <= 1e-6 * float(out["host"][1].abs().max())
        monkeypatch.setenv("DMNERF_INS_ASSIGN", "device")
        roc, nv = ins_assignment(cu(pred.numpy()), cu(lab.numpy()), k)
        assert int(nv) == len(label_values) and int((roc >= 0).sum()) == len(label_values)
    monkeypatch.setenv("DMNERF_INS_ASSIGN", "device")
    p = cu(pred.numpy()).requires_grad_(True)
    labd = cu(lab.numpy()).to(torch.int32)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        parts = ins_criterion(p, labd, k)
        parts[0].backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.isfinite(p.grad).all()


def test_instance_loss_rejected_labels_are_reported_on_the_next_call():
    """Labels the device ranking cannot take (>= 65536, negative, or more distinct labels than channels): that call's loss is NaN
    and its gradient zero -- nothing is read back -- and the NEXT ins_criterion call raises."""
    from dmnerf_b200.evaluator import ins_criterion
    gen = torch.Generator().manual_seed(2)
    pred = torch.sigmoid(torch.randn(128, 6, generator=gen))
    for lab in (torch.randint(0, 6, (128,), generator=gen) + 70000, torch.randint(0, 6, (128,), generator=gen) - 3,
                torch.arange(128) % 9):
        p = cu(pred.numpy()).requires_grad_(True)
        parts = ins_criterion(p, cu(lab.numpy()), 6)
        parts[0].backward()
        assert torch.isnan(parts[0]).all() and float(p.grad.abs().max()) == 0.0
        torch.cuda.synchronize()
        with pytest.raises(RuntimeError, match="earlier call"):
            ins_criterion(p, cu((torch.arange(128) % 6).numpy()), 6)
    parts = ins_criterion(cu(pred.numpy()), cu((torch.arange(128) % 6).numpy()), 6)       # the word was cleared: back to normal
    assert torch.isfinite(parts[0]).all()


def test_ray_selection_generates_only_the_selected_rays(golden_dir):
    """get_select_full / get_select_crop (helpers.py:64-111) natively: same numpy draws, rays bit-identical to the rows of the
    full get_rays_k grid, colours / labels gathered at the same pixels."""
    from dmnerf_b200.helpers import get_select_full, get_select_crop, get_rays_k
    wl = synth.workload("dmsr_study")
    H, W = 96, 128
    K = synth.dmsr_intrinsics(H, W)
    pose = cu(wl["c2w"])
    gen = torch.Generator().manual_seed(5)
    rgb = torch.rand(H, W, 3, generator=gen).to(DEV)
    lab = torch.randint(0, 13, (H, W), generator=gen).to(torch.int16).to(DEV)
    ro, rd = get_rays_k(H, W, K, pose)
    np.random.seed(11)
    expect = np.random.choice(H * W, size=[1024], replace=False)
    np.random.seed(11)
    tc, ti, rays = get_select_full(rgb, pose, K, lab, 1024)
    e = torch.from_numpy(expect).to(DEV)
    assert torch.equal(rays[0], ro.reshape(-1, 3)[e]) and torch.equal(rays[1], rd.reshape(-1, 3)[e])
    assert torch.equal(tc, rgb.reshape(-1, 3)[e]) and torch.equal(ti, lab.reshape(-1)[e])
    # crop variant: 30 % labelled pixels last, the rest from the crop mask, in the reference's draw order
    crop = np.zeros((H, W), dtype=np.int64); crop[8:80, 10:100] = 1
    ins_index = np.flatnonzero((crop.reshape(-1) == 1) & (np.arange(H * W) % 7 == 0))
    np.random.seed(12)
    n_ins = int(1000 * 0.3)
    labeled = ins_index[np.random.choice(len(ins_index), size=[n_ins], replace=False)]
    crop_idx = np.where(crop.reshape(-1) == 1)[0]
    n_un = len(set(crop_idx) - set(labeled))
    unl = crop_idx[np.random.choice(n_un, size=[1000 - n_ins], replace=False)]
    np.random.seed(12)
    tc, ti, rays, got_n = get_select_crop(rgb, pose, K, lab, ins_index, crop, 1000)
    sel = torch.from_numpy(np.concatenate([unl, labeled])).to(DEV)
    assert got_n == n_ins and rays.shape == (2, 1000, 3)
    assert torch.equal(rays[1], rd.reshape(-1, 3)[sel]) and torch.equal(tc, rgb.reshape(-1, 3)[sel])
    assert torch.equal(ti, lab.reshape(-1)[torch.from_numpy(labeled).to(DEV)])


def test_device_side_pixel_selection_and_device_resident_pose(monkeypatch):
    """DMNERF_SELECT=device: N distinct in-range pixels from the keyed-bijection kernel (every pixel reachable, seeds differ,
    roughly uniform), rays bit-identical to the full grid at those pixels; and get_rays_at reads a strided device pose without
    synchronising."""
    from dmnerf_b200.helpers import get_select_full, get_rays_k, get_rays_at, select_pixels
    wl = synth.workload("dmsr_study")
    H, W = 480, 640
    K = wl["K"]
    pose44 = torch.eye(4, device=DEV)
    pose44[:3, :4] = cu(wl["c2w"])[:3, :4]
    a = select_pixels(H, W, 1024, DEV, seed=5).cpu().numpy()
    b = select_pixels(H, W, 1024, DEV, seed=6).cpu().numpy()
    assert len(set(a.tolist())) == 1024 and a.min() >= 0 and a.max() < H * W and len(set(a.tolist()) & set(b.tolist())) < 40
    full = select_pixels(37, 41, 37 * 41, DEV, seed=9).cpu().numpy()               # the whole image: a permutation
    assert sorted(full.tolist()) == list(range(37 * 41))
    hist = np.zeros(16)
    for s in range(64):
        hist += np.bincount(select_pixels(H, W, 4096, DEV, seed=1000 + s).cpu().numpy() * 16 // (H * W), minlength=16)
    assert np.abs(hist / hist.sum() - 1 / 16).max() < 0.004                       # 262 144 draws: sigma of a bin share = 0.0005
    assert select_pixels(H, W, 0, DEV, seed=1).shape == (0,)
    ro, rd = get_rays_k(H, W, K, pose44[:3, :4])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        pix = select_pixels(H, W, 777, DEV, seed=3)
        o2, d2 = get_rays_at(H, W, K, pose44, pix)                                # [4,4] device pose, rows 4 floats apart
        o3, d3 = get_rays_at(H, W, K, pose44[:3, :4], pix)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.equal(d2, rd.reshape(-1, 3)[pix]) and torch.equal(o2, ro.reshape(-1, 3)[pix])
    assert torch.equal(d3, d2) and torch.equal(o3, o2)
    monkeypatch.setenv("DMNERF_SELECT", "device")
    import dmnerf_b200.helpers as helpers_mod
    drawn = []
    real = helpers_mod.select_pixels
    monkeypatch.setattr(helpers_mod, "select_pixels", lambda *a, **k: drawn.append(real(*a, **k)) or drawn[-1])
    gen = torch.Generator().manual_seed(5)
    rgb = torch.rand(H, W, 3, generator=gen).to(DEV)
    lab = torch.randint(0, 13, (H, W), generator=gen).to(torch.int16).to(DEV)
    np.random.seed(4)
    tc, ti, rays = get_select_full(rgb, pose44[:3, :4], K, lab, 1024)
    np.random.seed(4)
    tc2, ti2, rays2 = get_select_full(rgb, pose44[:3, :4], K, lab, 1024)
    assert rays.shape == (2, 1024, 3) and tc.shape == (1024, 3) and ti.shape == (1024,) and len(drawn) == 2
    assert not torch.equal(drawn[0], drawn[1])                                    # the call counter moves the permutation on
    p0 = drawn[0]
    assert len(set(p0.tolist())) == 1024
    assert torch.equal(rays[1], rd.reshape(-1, 3)[p0]) and torch.equal(rays[0], ro.reshape(-1, 3)[p0])
    assert torch.equal(tc, rgb.reshape(-1, 3)[p0]) and torch.equal(ti, lab.reshape(-1)[p0])


def test_reference_training_iteration_through_the_dropin_imports():
    """One iteration of train_dmsr.py:23-64 written against the drop-in `networks` package exactly as the reference script
    imports it (ray selection -> dm_nerf -> MSE + Hungarian instance loss + emptiness penalizer -> backward -> Adam), every
    stage on the native kernels (launch counter) and making progress over a few steps."""
    import sys
    drop = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dm-nerf_b200", "dropin")
    saved = {k: v for k, v in sys.modules.items() if k == "networks" or k.startswith("networks.")}
    for k in saved:
        del sys.modules[k]
    sys.path.insert(0, drop)
    try:
        from networks.render import dm_nerf
        from networks.dm_nerf import get_embedder, DM_NeRF
        from networks.penalizer import ins_penalizer
        from networks.helpers import get_select_full, z_val_sample
        from networks.evaluator import ins_criterion, img2mse, mse2psnr
        import networks.render as nr_mod
        assert "dmnerf_b200" in nr_mod.dm_nerf.__module__
        H, W, ins_num, n_train = 48, 64, 13, 512
        wl = synth.workload("dmsr_study")
        K = synth.dmsr_intrinsics(H, W)
        pose = cu(wl["c2w"])
        gen = torch.Generator().manual_seed(9)
        gt_rgb = torch.rand(H, W, 3, generator=gen).to(DEV)
        gt_label = (torch.arange(H * W).reshape(H, W) * 7 // (H * W)).to(torch.int16).to(DEV)      # 7 objects present
        torch.manual_seed(0); np.random.seed(0)
        pe, _ = get_embedder(10); ve, _ = get_embedder(4)
        mc, mf = DM_NeRF(8, 256, 63, 27, [4], ins_num).to(DEV), DM_NeRF(8, 256, 63, 27, [4], ins_num).to(DEV)
        mc.train(); mf.train()
        opt = torch.optim.Adam(list(mc.parameters()) + list(mf.parameters()), lr=5e-4, betas=(0.9, 0.999))
        args = types.SimpleNamespace(perturb=0.0, N_importance=128, is_train=True, N_ins=None, N_train=n_train, near=4.0, far=15.0,
                                     N_samples=64, ins_num=ins_num, tolerance=0.05, deta_w=0.05, penalize=True)
        z_val_coarse = z_val_sample(args.N_train, args.near, args.far, args.N_samples, device=DEV)
        before = _lib.launch_count()
        losses, mses = [], []
        for it in range(8):
            np.random.seed(1)                                   # same pixels every iteration: the colour loss must go down
            target_c, target_i, batch_rays = get_select_full(gt_rgb, pose, K, gt_label, args.N_train)
            all_info = dm_nerf(batch_rays, pe, ve, mc, mf, z_val_coarse, args)
            rgb_loss = img2mse(all_info["rgb_coarse"], target_c) + img2mse(all_info["rgb_fine"], target_c)
            ins_c = ins_criterion(all_info["ins_coarse"], target_i, args.ins_num)
            ins_f = ins_criterion(all_info["ins_fine"], target_i, args.ins_num)
            total = ins_c[0] + ins_f[0] + rgb_loss
            total = total + ins_penalizer(all_info["raw_coarse"], all_info["z_vals_coarse"], all_info["depth_coarse"], batch_rays[1], args) \
                + ins_penalizer(all_info["raw_fine"], all_info["z_vals_fine"], all_info["depth_fine"], batch_rays[1], args)
            opt.zero_grad()
            total.backward()
            opt.step()
            assert torch.isfinite(mse2psnr(img2mse(all_info["rgb_fine"], target_c))).all()
            assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in list(mc.parameters()) + list(mf.parameters()))
            assert float(mf.ins_linear.weight.grad.abs().max()) > 0 and float(mc.mlps[0].weight.grad.abs().max()) > 0
            losses.append(float(total.sum()))
            mses.append(float(rgb_loss))
        assert _lib.launch_count() - before > 60          # ray selection, render, losses, backward: all native launches
        assert np.isfinite(losses).all()
        # the instance terms re-match every step (Hungarian) and may wander at first; the colour term has a fixed target
        assert min(mses[4:]) < mses[0], (mses, losses)
    finally:
        sys.path.remove(drop)
        for k in [k for k in sys.modules if k == "networks" or k.startswith("networks.")]:
            del sys.modules[k]
        sys.modules.update(saved)


def _noisy_oracle_grads(w, x, G, amp, seed):
    """Oracle autograd with zero-mean noise of relative amplitude `amp` (x the layer's rms) injected into every pre-activation:
    a stand-in for ANY forward arithmetic that is accurate to ~amp (e.g. the split-bf16 tensor-core products)."""
    p = O.to_torch(w)
    for v in p.values():
        v.requires_grad_(True)
    gen = torch.Generator().manual_seed(seed)
    real_lin = O._lin

    def noisy(pp, name, inp):
        out = real_lin(pp, name, inp)
        if out.shape[-1] >= 128:                       # hidden layers (the ReLU inputs); the narrow heads stay exact
            out = out + (amp * out.detach().pow(2).mean().sqrt()) * torch.randn(out.shape, generator=gen)
        return out

    O._lin = noisy
    try:
        (O.mlp_forward(p, x) * G).sum().backward()
    finally:
        O._lin = real_lin
    return {k: v.grad.numpy() for k, v in p.items()}


def test_tensor_core_gradient_deviation_is_relu_flip_sensitivity():
    """With the tensor-core forward the parameter gradients deviate from the exact ones by up to ~5e-3 relative L2 although every
    activation is accurate to ~1e-5: units sitting within that distance of zero get the other ReLU branch.  This is a property of
    the loss surface, not of the kernels: injecting 1e-5 noise into the ORACLE's pre-activations moves its own gradients by the
    same amount, and the native path must stay inside a small multiple of that band."""
    m, ins_num = 4096, 13
    w = synth.make_weights(21, ins_num)
    gen = torch.Generator().manual_seed(9)
    pts = torch.rand(m, 3, generator=gen) * 6 - 3
    vd = torch.randn(m, 3, generator=gen)
    vd = vd / vd.norm(dim=-1, keepdim=True)
    x = torch.cat([O.embed(pts, 10), O.embed(vd, 4)], -1)
    G = torch.randn(m, 4 + ins_num + 1, generator=gen)
    exact = _noisy_oracle_grads(w, x, G, 0.0, 0)
    noisy = [_noisy_oracle_grads(w, x, G, 1e-5, s) for s in (1, 2)]
    net = model_from_weights(w, DEV).train()
    y = net(x.to(DEV), impl=_lib.IMPL_UMMA)
    (y * G.to(DEV)).sum().backward()
    from dmnerf_b200.engine import get_context
    get_context(torch.device(DEV)).sync_check()
    worst = 0.0
    for k, prm in net.named_parameters():
        if exact[k].size < 128:
            continue                                     # tiny bias vectors of the heads: relL2 is not meaningful
        ours = rel_l2(prm.grad.cpu().numpy(), exact[k])
        band = max(rel_l2(n[k], exact[k]) for n in noisy)
        worst = max(worst, ours)
        print("%-34s relL2 ours %.2e   oracle with 1e-5 activation noise %.2e" % (k, ours, band))
        assert ours <= 6.0 * band + 2e-4, (k, ours, band)
    assert worst <= 2e-2
