"""CPU: the oracle (oracle/dmnerf_oracle.py) against the fixtures written by oracle/make_golden.py from
the unmodified reference.  On the machine that generated them the match is bit-exact; elsewhere the
host BLAS may round differently, hence the small tolerances (stage-wise, teacher-forced inputs)."""
import os

import numpy as np
import pytest
import torch

from oracle import dmnerf_oracle as O
from dmnerf_b200 import synth

RTOL, ATOL = 2e-5, 2e-6


def load(golden_dir, name):
    return dict(np.load(os.path.join(golden_dir, name)))


def close(a, b, rtol=RTOL, atol=ATOL):
    np.testing.assert_allclose(a.detach().numpy() if torch.is_tensor(a) else a, b, rtol=rtol, atol=atol)


def test_embed(golden_dir):
    g = load(golden_dir, "embed.npz")
    x = torch.from_numpy(g["x"])
    close(O.embed(x, 10), g["pos"])
    close(O.embed(x / x.norm(dim=-1, keepdim=True), 4), g["dir"])
    assert g["pos"].shape[1] == 63 and g["dir"].shape[1] == 27


def test_mlp(golden_dir):
    for ins_num in (13, 59):
        g = load(golden_dir, "mlp_ins%d.npz" % ins_num)
        w = O.to_torch(synth.make_weights(int(g["seed"]), ins_num))
        y = O.mlp_forward(w, torch.from_numpy(g["x"]))
        assert y.shape[1] == 4 + ins_num + 1
        close(y, g["y"], rtol=1e-4, atol=1e-5)


def test_composite(golden_dir):
    g = load(golden_dir, "composite.npz")
    rgb, w, d, ins, acc = O.composite(torch.from_numpy(g["raw"]), torch.from_numpy(g["z"]), torch.from_numpy(g["rays_d"]))
    close(rgb, g["rgb"]); close(w, g["weights"]); close(d, g["depth"]); close(ins, g["ins"])
    close(acc, g["weights"].sum(-1), rtol=1e-5)
    assert float(w[0].abs().max()) == 0.0            # empty ray
    assert float(w[1, :4].sum()) > 0.99              # (nearly) opaque at the first samples


def test_sample_pdf(golden_dir):
    g = load(golden_dir, "sample_pdf.npz")
    b, w = torch.from_numpy(g["bins"]), torch.from_numpy(g["weights"])
    close(O.sample_pdf(b, w, 128, det=True), g["det"], rtol=1e-5, atol=1e-5)
    close(O.sample_pdf(b, w, 128, det=False, u=torch.from_numpy(g["u"])), g["rnd"], rtol=1e-5, atol=1e-5)


def test_rays_and_z(golden_dir):
    g = load(golden_dir, "rays.npz")
    o, d = O.get_rays_k(480, 640, torch.from_numpy(g["K"]), torch.from_numpy(g["c2w"]))
    close(d.reshape(-1, 3)[g["idx"]], g["rays_d"]); close(o.reshape(-1, 3)[g["idx"]], g["rays_o"])
    close(O.z_val_sample(3, 4.0, 15.0, 64)[1], g["z"], rtol=0, atol=0)
    close(O.z_val_sample(3, 0.0, 6.5, 64)[2], g["z_replica"], rtol=0, atol=0)
    wl = synth.workload("dmsr_study")                # numpy twin used by bench/tests
    close(wl["rays_d"][g["idx"]], g["rays_d"], rtol=1e-6, atol=1e-6)


def _render_case(golden_dir, tag):
    g = load(golden_dir, "render_%s.npz" % tag)
    ins_num = int(g["ins_num"])
    pc = O.to_torch(synth.make_weights(int(g["seed_coarse"]), ins_num))
    pf = O.to_torch(synth.make_weights(int(g["seed_fine"]), ins_num))
    ro, rd = torch.from_numpy(g["rays_o"]), torch.from_numpy(g["rays_d"])
    zc = O.z_val_sample(ro.shape[0], float(g["near"]), float(g["far"]), 64)
    return g, pc, pf, ro, rd, zc


def test_render_inference(golden_dir):
    for tag in ("study", "room0"):
        g, pc, pf, ro, rd, zc = _render_case(golden_dir, tag)
        with torch.no_grad():
            out = O.render(ro, rd, pc, pf, zc, perturb=0.0)
        for k in ("rgb_fine", "ins_fine", "z_vals_fine", "raw_fine", "raw_coarse", "rgb_coarse", "ins_coarse",
                  "z_vals_coarse", "depth_fine", "depth_coarse"):
            close(out[k], g["det_" + k], rtol=2e-3, atol=2e-3)     # end-to-end: ill-conditioned (SURVEY 7)
        z = out["z_vals_fine"]
        assert bool((z[:, 1:] >= z[:, :-1]).all())
        assert float(out["acc_fine"].max()) <= 1.0 + 1e-5


def test_hier_sample_restates_render(golden_dir):
    """O.hier_sample fed the render's own coarse depths and weights gives the render's fine depths bit for bit, deterministic
    and with given uniforms (the GPU sampler tests compare against it)."""
    g, pc, pf, ro, rd, zc = _render_case(golden_dir, "study")
    with torch.no_grad():
        for perturb, t_rand, u in ((0.0, None, None), (1.0, torch.from_numpy(g["t_rand"]), torch.from_numpy(g["u"]))):
            out = O.render(ro, rd, pc, pf, zc, perturb=perturb, t_rand=t_rand, u=u)
            zf = O.hier_sample(out["z_vals_coarse"], out["weights_coarse"], 128, det=perturb == 0.0, u=u)
            assert zf.shape == out["z_vals_fine"].shape and torch.equal(zf, out["z_vals_fine"])


def test_render_train_and_grads(golden_dir):
    g, pc, pf, ro, rd, zc = _render_case(golden_dir, "study")
    for d in (pc, pf):
        for v in d.values():
            v.requires_grad_(True)
    out = O.render(ro, rd, pc, pf, zc, perturb=1.0, t_rand=torch.from_numpy(g["t_rand"]), u=torch.from_numpy(g["u"]),
                   is_train=True)
    loss = O.train_loss(out, torch.from_numpy(g["target"]))
    close(loss, g["loss"], rtol=1e-4)
    loss.backward()
    for nm, d in (("coarse", pc), ("fine", pf)):
        for k, v in d.items():
            ref = g["grad_%s_%s" % (nm, k)]
            got = v.grad if v.grad is not None else torch.zeros_like(v)
            if k.endswith("weight"):
                got = got[::8, ::8]
            scale = max(float(np.abs(ref).max()), 1e-8)
            assert float((got - torch.from_numpy(ref)).abs().max()) <= 2e-3 * scale + 1e-9, (nm, k)
    # detach topology (SURVEY 3.3): the instance terms never reach the trunk through ins_feature_linear's input
    assert pc["mlps.0.weight"].grad is not None


def test_fp64_twin_noise_floor(golden_dir):
    """The fp32 oracle vs its own fp64 twin: the yard-stick for what 'parity' can mean stage-wise."""
    g = load(golden_dir, "mlp_ins13.npz")
    w = synth.make_weights(int(g["seed"]), 13)
    y32 = O.mlp_forward(O.to_torch(w), torch.from_numpy(g["x"]))
    y64 = O.mlp_forward(O.to_torch(w, torch.float64), torch.from_numpy(g["x"]).double())
    rel = float((y32.double() - y64).norm() / y64.norm())
    assert rel < 5e-6


def test_penalizer(golden_dir):
    """Oracle emptiness penalizer (networks/penalizer.py:5-62) against the reference's loss and raw-gradient."""
    g = load(golden_dir, "penalizer.npz")
    for tag in ("a", "b"):
        raw = torch.from_numpy(g["raw_" + tag]).clone().requires_grad_(True)
        loss = O.ins_penalizer(raw, torch.from_numpy(g["z_" + tag]), torch.from_numpy(g["depth_" + tag]),
                               torch.from_numpy(g["rays_d_" + tag]), float(g["tolerance"]), float(g["deta_w"]))
        loss.sum().backward()
        close(loss, g["loss_" + tag])
        close(raw.grad, g["grad_" + tag], atol=1e-9)


def test_evaluator(golden_dir):
    """Oracle Hungarian-matched instance loss (networks/evaluator.py:19-74) against the reference's loss parts, cost matrices,
    assignment and gradient w.r.t. the rendered instance map."""
    g = load(golden_dir, "evaluator.npz")
    for tag in ("a", "b", "c"):
        k = int(g["k_" + tag])
        pred = torch.from_numpy(g["pred_" + tag]).clone().requires_grad_(True)
        lab = torch.from_numpy(g["labels_" + tag])
        parts = O.ins_criterion(pred, lab, k)
        parts[0].sum().backward()
        close(torch.stack([x.detach().float().sum() for x in parts]), g["loss_" + tag])
        close(pred.grad, g["grad_" + tag], atol=1e-9)
        valid = torch.unique(lab)
        gt = torch.zeros(lab.shape[0], k)
        gt[:, :len(valid)] = torch.nn.functional.one_hot(lab.long())[..., valid.long()]
        ce, siou, _, cols = O.hungarian(pred.detach(), gt, len(valid), k)
        close(ce, g["cost_ce_" + tag]); close(siou, g["cost_siou_" + tag])
        assert list(cols) == list(g["order_col_" + tag])


def test_manipulator(golden_dir):
    """Oracle edit pipeline (networks/manipulator.py:18-205) against the reference run stored in manipulator.npz."""
    g = load(golden_dir, "manipulator.npz")
    ins_num = int(g["ins_num"])
    wc, wf = synth.make_weights(int(g["seed_c"]), ins_num), synth.make_weights(int(g["seed_f"]), ins_num)
    wc["ins_linear.weight"], wc["ins_linear.bias"] = g["ins_w_c"], g["ins_b_c"]
    wf["ins_linear.weight"], wf["ins_linear.bias"] = g["ins_w_f"], g["ins_b_f"]
    t = torch.from_numpy
    labels = [int(v) for v in g["labels"]]
    with torch.no_grad():
        out = O.exchanger(t(g["ex_ori_raw"]), [t(x) for x in g["ex_tar_raws"]], t(g["ex_acc_o"]), [t(x) for x in g["ex_acc_t"]], labels)
        assert torch.equal(out[0], t(g["ex_out_raw"])) and torch.equal(out[2], t(g["ex_out_label"]))
        assert torch.equal(out[3], t(g["ex_out_tar_label"]))
        res = O.manipulator(O.to_torch(wc), O.to_torch(wf), t(g["ori"]), [t(x) for x in g["f_tar"]], int(g["n_samples"]),
                            int(g["n_importance"]), float(g["near"]), float(g["far"]), labels, us=[t(u) for u in g["us"]])
    close(res[2], g["tar_rgb"], rtol=1e-4, atol=1e-5)
    # discrete decisions inside: bulk agreement (bit-exact on the generating machine)
    for got, key in ((res[0], "final_rgb"), (res[1], "final_ins"), (res[3], "tar_ins_accum")):
        assert (np.abs(got.numpy() - g[key]).max(-1) <= 1e-3).mean() >= 0.9, key


def test_oracle_domain_properties():
    """Size-independent properties of the path (SURVEY.md 8c), on the oracle: sum of weights <= 1, the merged depths are sorted
    and stay inside [near, far], deterministic importance sampling is monotone, the instance map lies in (0, 1)."""
    gen = torch.Generator().manual_seed(3)
    for n, s in ((5, 64), (3, 17)):
        raw = torch.randn(n, s, 18, generator=gen) * 2
        z = O.z_val_sample(n, 4.0, 15.0, s)
        rd = torch.randn(n, 3, generator=gen)
        rgb, w, depth, ins, acc = O.composite(raw, z, rd)
        assert float(acc.max()) <= 1.0 + 1e-6 and float(w.min()) >= 0.0
        assert float(ins.min()) > 0.0 and float(ins.max()) < 1.0
        mid = .5 * (z[..., 1:] + z[..., :-1])
        zs = O.sample_pdf(mid, w[..., 1:-1], 40, det=True)
        assert bool((zs[..., 1:] >= zs[..., :-1] - 1e-6).all())
        zf = torch.sort(torch.cat([z, zs], -1), -1).values
        assert float(zf.min()) >= 4.0 - 1e-5 and float(zf.max()) <= 15.0 + 1e-5


def test_assignment_restatement_is_scipys_algorithm():
    """oracle/lsap.py (the shortest-augmenting-path solver scipy implements; the reference calls scipy at evaluator.py:45) against
    the installed scipy: the SAME columns on random, tie-heavy integer, constant and duplicate-column matrices -- for the
    column-by-column form and for the order-free arg-min form the device kernel uses."""
    from scipy.optimize import linear_sum_assignment
    from oracle import lsap
    n = 0
    for c in lsap.tie_heavy_cases(400, 24, seed=7):
        rows, cols = linear_sum_assignment(c)
        r1, c1 = lsap.lsap_sequential(c)
        r2, c2 = lsap.lsap_lane_parallel(c)
        assert np.array_equal(r1, rows) and np.array_equal(c1, cols), c.shape
        assert np.array_equal(c2, cols), c.shape
        n += 1
    assert n == 400
    big = next(iter(lsap.tie_heavy_cases(1, 94, seed=11)))
    assert np.array_equal(lsap.lsap_lane_parallel(big)[1], linear_sum_assignment(big)[1])
    with pytest.raises(ValueError):
        lsap.lsap_sequential(np.full((2, 2), np.inf))
