"""GPU: edge cases of the call surface -- empty / ragged batches, per-ray coarse depths, the ScanNet N_ins slice,
the widest object head, keep-all-instance-channels, no_grad + perturb through dm_nerf, non-contiguous inputs."""
import os
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from dmnerf_b200 import synth, _lib
from dmnerf_b200.testing import make_models, model_from_weights

DEV = "cuda"


def _rays(n, name="dmsr_study"):
    wl = synth.workload(name)
    sel = np.linspace(0, 307199, max(n, 1)).astype(np.int64)[:n]
    return wl, torch.from_numpy(wl["rays_o"][sel]).to(DEV), torch.from_numpy(wl["rays_d"][sel]).to(DEV)


def test_empty_batch_and_single_ray():
    from dmnerf_b200.render import render_rays
    wl, ro, rd = _rays(3)
    nc, nf, _, _ = make_models(1, 2, 13, DEV)
    z = torch.linspace(4, 15, 64, device=DEV)
    with torch.no_grad():
        for want_raw in (False, True):
            out = render_rays(ro[:0], rd[:0], nc, nf, z, want_raw=want_raw)
            assert out["rgb_fine"].shape == (0, 3) and out["ins_fine"].shape == (0, 13)
            one = render_rays(ro[:1], rd[:1], nc, nf, z, want_raw=want_raw)
            three = render_rays(ro, rd, nc, nf, z, want_raw=want_raw)
            assert torch.isfinite(one["rgb_fine"]).all()
            if not want_raw:
                assert torch.equal(one["rgb_fine"], three["rgb_fine"][:1])       # rays are independent units


@pytest.mark.parametrize("want_raw", [False, True])
def test_per_ray_coarse_depths_match_shared_row(want_raw):
    """z_vals_coarse may be a real [N,S] tensor (reference: any tensor broadcastable in render.py:49) or the stride-0
    expand that z_val_sample returns: both must give the same render."""
    from dmnerf_b200.render import render_rays
    from dmnerf_b200.helpers import z_val_sample
    wl, ro, rd = _rays(130)
    nc, nf, _, _ = make_models(1, 2, 13, DEV)
    zs = z_val_sample(130, wl["near"], wl["far"], 64, device=DEV)
    with torch.no_grad():
        a = render_rays(ro, rd, nc, nf, zs, want_raw=want_raw)
        b = render_rays(ro, rd, nc, nf, zs.contiguous(), want_raw=want_raw)          # materialised [N,S]
    for k in ("rgb_fine", "depth_fine", "ins_fine", "rgb_coarse"):
        assert torch.equal(a[k], b[k]), k


def test_per_ray_coarse_depths_with_too_few_rows_are_rejected():
    """A per-ray z_vals_coarse with fewer rows than rays is an error for inference and training alike; training raises
    before its first launch instead of reading past the end of the depths."""
    from dmnerf_b200.render import dm_nerf, render_rays
    from dmnerf_b200.embedder import get_embedder
    wl, ro, rd = _rays(130)
    nc, nf, _, _ = make_models(1, 2, 13, DEV)
    z = torch.linspace(wl["near"], wl["far"], 64, device=DEV).repeat(129, 1)
    with torch.no_grad(), pytest.raises(RuntimeError, match="129 rows for 130 rays"):
        render_rays(ro, rd, nc, nf, z)
    args = types.SimpleNamespace(perturb=1.0, N_importance=128)
    before = _lib.launch_count()
    with pytest.raises(RuntimeError, match="129 rows for 130 rays"):
        dm_nerf(torch.stack([ro, rd], 0), get_embedder(10)[0], get_embedder(4)[0], nc, nf, z, args)
    assert _lib.launch_count() == before


def test_scannet_n_ins_slice_and_perturb_without_grad():
    """render.py:88-90: with args.is_train and args.N_ins only the last N_ins rays keep instance maps; perturb > 0 under
    no_grad (manipulator-style) must consume the two uniform draws in the reference's order."""
    from dmnerf_b200.render import dm_nerf
    from dmnerf_b200.embedder import get_embedder
    from dmnerf_b200.helpers import z_val_sample
    wl, ro, rd = _rays(64)
    nc, nf, _, _ = make_models(1, 2, 13, DEV)
    pe, ve = get_embedder(10)[0], get_embedder(4)[0]
    zc = z_val_sample(64, wl["near"], wl["far"], 64, device=DEV)
    args = types.SimpleNamespace(perturb=1.0, N_importance=128, is_train=True, N_ins=20)
    with torch.no_grad():
        torch.manual_seed(11)
        out = dm_nerf(torch.stack([ro, rd], 0), pe, ve, nc, nf, zc, args)
        torch.manual_seed(11)
        t_rand, u = torch.rand((64, 64), device=DEV), torch.rand((64, 128), device=DEV)
        from dmnerf_b200.render import render_rays
        ref = render_rays(ro, rd, nc, nf, zc, perturb=1.0, t_rand=t_rand, u=u, want_raw=False)
    assert out["ins_fine"].shape == (20, 13) and out["ins_coarse"].shape == (20, 13) and out["rgb_fine"].shape == (64, 3)
    assert torch.equal(out["rgb_fine"], ref["rgb_fine"]) and torch.equal(out["ins_fine"], ref["ins_fine"][-20:])
    zf = out["z_vals_fine"]                                             # lazily materialised per-sample outputs
    assert zf.shape == (64, 192) and bool((zf[:, 1:] >= zf[:, :-1]).all())


def test_widest_object_head_and_keep_all_channels():
    from dmnerf_b200.render import render_rays
    wl, ro, rd = _rays(70)
    nc, nf, _, _ = make_models(5, 6, 127, DEV)                           # ins_num + 1 = 128 output columns: the maximum
    z = torch.linspace(4, 15, 64, device=DEV)
    with torch.no_grad():
        fused = render_rays(ro, rd, nc, nf, z, want_raw=False)
        staged = render_rays(ro, rd, nc, nf, z, want_raw=True)
        keep = render_rays(ro, rd, nc, nf, z, want_raw=False, keep_all_ins=True)
    assert fused["ins_fine"].shape == (70, 127) and staged["raw_fine"].shape == (70, 192, 132) and keep["ins_fine"].shape == (70, 128)
    np.testing.assert_allclose(fused["ins_coarse"].cpu().numpy(), staged["ins_coarse"].cpu().numpy(), rtol=1e-4, atol=5e-6)
    np.testing.assert_allclose(keep["ins_fine"][:, :-1].cpu().numpy(), fused["ins_fine"].cpu().numpy(), rtol=0, atol=0)
    with pytest.raises(ValueError):
        from dmnerf_b200.model import DM_NeRF
        DM_NeRF(8, 256, 63, 27, [4], 128)


def test_non_contiguous_and_batched_inputs():
    from dmnerf_b200.render import render_train
    from dmnerf_b200.embedder import get_embedder
    from dmnerf_b200.helpers import sample_pdf
    raw = torch.randn(6, 40, 18 * 2, device=DEV)[..., ::2]                # non-contiguous channel stride
    z = torch.sort(torch.rand(6, 40, device=DEV) * 5 + 1).values
    rd = torch.randn(6, 3, device=DEV)
    a = render_train(raw, z, rd)
    b = render_train(raw.contiguous(), z, rd)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    x = torch.randn(2, 5, 7, 3, device=DEV)                               # leading dims are preserved
    assert get_embedder(10)[0].embed(x).shape == (2, 5, 7, 63)
    bins = torch.sort(torch.rand(2, 3, 63, device=DEV)).values
    s = sample_pdf(bins, torch.rand(2, 3, 62, device=DEV), 16, det=True)
    assert s.shape == (2, 3, 16) and bool((s[..., 1:] >= s[..., :-1] - 1e-6).all())
    assert isinstance(get_embedder(0, -1)[0], torch.nn.Identity)


def test_render_frame_driver_matches_explicit_rays():
    """dmnerf_render_frame_host (render_test's per-camera loop, tester.py:55-76): rays generated on the device from K / c2w,
    coarse depths from near / far -- identical (bitwise: same kernels, same inputs) to get_rays_k + z_val_sample + dm_nerf on
    explicit rays; a pixel range renders the matching slice."""
    import types
    from dmnerf_b200 import synth
    from dmnerf_b200.testing import make_models
    from dmnerf_b200.render import render_frame, dm_nerf
    from dmnerf_b200.helpers import get_rays_k, z_val_sample
    from dmnerf_b200.embedder import get_embedder
    wl = synth.workload("dmsr_study")
    nc, nf, _, _ = make_models(3, 4, 13, "cuda")
    H, W = 12, 20
    K = np.array(wl["K"], dtype=np.float32).copy()
    K[0, 2], K[1, 2] = W / 2, H / 2
    c2w = torch.from_numpy(np.asarray(wl["c2w"], dtype=np.float32))
    near, far = float(wl["near"]), float(wl["far"])
    with torch.no_grad():
        fr = render_frame(H, W, K, c2w, near, far, nc, nf)
        ro, rd = get_rays_k(H, W, K, c2w.cuda())
        rays = torch.stack([ro.reshape(-1, 3), rd.reshape(-1, 3)], 0)
        args = types.SimpleNamespace(perturb=0.0, N_importance=128, is_train=False, N_ins=None)
        ref = dm_nerf(rays, get_embedder(10)[0], get_embedder(4)[0], nc, nf, z_val_sample(H * W, near, far, 64, device="cuda"), args)
        part = render_frame(H, W, K, c2w, near, far, nc, nf, pixel_range=(37, 101))
    assert fr["rgb"].shape == (H, W, 3) and fr["ins"].shape == (H, W, 13) and fr["depth"].shape == (H, W)
    assert torch.equal(fr["rgb"].reshape(-1, 3), ref["rgb_fine"].cpu())
    assert torch.equal(fr["ins"].reshape(-1, 13), ref["ins_fine"].cpu())
    assert torch.equal(fr["depth"].reshape(-1), ref["depth_fine"].cpu())
    assert torch.equal(part["rgb"], ref["rgb_fine"].cpu()[37:138]) and torch.equal(part["acc"], fr["acc"].reshape(-1)[37:138])


def test_host_entry_point_in_parts_is_bitwise_the_single_launch():
    """dmnerf_render_forward_host on >= 131 072 rays renders the batch in four parts whose copies overlap the neighbouring
    parts' kernels (second stream): same bits as the device-resident single launch, odd ray count, per-ray depth rows
    (z_row_stride != 0) and the shared row (stride 0), a small batch (single part) through the same call, an object
    selection (io.edit->keep) against dmnerf_render_forward with the same mask, and the fp16 preview network."""
    import ctypes as C
    from dmnerf_b200.testing import make_models
    from dmnerf_b200.engine import get_context
    from dmnerf_b200.objects import object_mask
    from dmnerf_b200.render import render_rays
    wl = synth.workload("dmsr_study")
    nc, nf, _, _ = make_models(5, 6, 13, "cuda")
    ctx = get_context(torch.device("cuda"))
    ctx.bind(0, nc); ctx.bind(1, nf)
    F16 = _lib.IMPL_UMMA_F16
    with torch.no_grad():                                               # pack the fp16 images outside the launch count
        render_rays(torch.from_numpy(wl["rays_o"][:2]).cuda(), torch.from_numpy(wl["rays_d"][:2]).cuda(), nc, nf,
                    torch.linspace(float(wl["near"]), float(wl["far"]), 64, device="cuda"), want_raw=False, impl=F16)
    cases = ((131073, False, None, 0), (131080, True, None, 0), (4097, False, None, 0), (131073, False, [0, 2, 3, 7, 13], 0),
             (131073, True, None, F16))
    for n, per_ray_z, keep, impl in cases:
        ro = torch.from_numpy(wl["rays_o"][:n]).contiguous().pin_memory()
        rd = torch.from_numpy(wl["rays_d"][:n]).contiguous().pin_memory()
        zrow = torch.linspace(float(wl["near"]), float(wl["far"]), 64)
        zc = (zrow[None].expand(n, 64) + 0.01 * torch.arange(n)[:, None] / n).contiguous() if per_ray_z else zrow.contiguous()
        zc = zc.pin_memory()
        out = {k: torch.full((n,) + shape, float("nan")).pin_memory() for k, shape in
               (("rgb_fine", (3,)), ("depth_fine", ()), ("acc_coarse", ()), ("ins_fine", (13,)))}
        io = _lib.RenderIO()
        io.rays_o, io.rays_d, io.z_coarse, io.z_row_stride = _lib.ptr(ro), _lib.ptr(rd), _lib.ptr(zc), (64 if per_ray_z else 0)
        for k, v in out.items():
            setattr(io, k, _lib.ptr(v))
        if keep is not None:
            words = _lib.keep_mask(object_mask(13, keep=keep))
            edit = _lib.Edit(keep=C.cast(words, C.POINTER(C.c_uint32)))
            io.edit = C.pointer(edit)
        before = _lib.launch_count()
        _lib.check(ctx.lib.dmnerf_render_forward_host(ctx.handle, io, n, 64, 128, 0, impl, ctx.stream()), "dmnerf_render_forward_host")
        launches = _lib.launch_count() - before
        assert launches == (4 if n >= 131072 else 1), launches
        with torch.no_grad():
            zdev = zc.cuda() if per_ray_z else zc.cuda()[None].expand(n, 64)
            ref = render_rays(ro.cuda(), rd.cuda(), nc, nf, zdev, N_importance=128, want_raw=False, keep_objects=keep,
                              impl=impl)
        for k, v in out.items():
            assert torch.equal(v, ref[k].cpu()), (n, keep, impl, k)


def _manip_setup(golden_dir):
    g = dict(np.load(os.path.join(golden_dir, "manipulator.npz")))
    ins_num = int(g["ins_num"])
    from dmnerf_b200.testing import model_from_weights
    wc, wf = synth.make_weights(int(g["seed_c"]), ins_num), synth.make_weights(int(g["seed_f"]), ins_num)
    wc["ins_linear.weight"], wc["ins_linear.bias"] = g["ins_w_c"], g["ins_b_c"]
    wf["ins_linear.weight"], wf["ins_linear.bias"] = g["ins_w_f"], g["ins_b_f"]
    return g, model_from_weights(wc, "cuda").eval(), model_from_weights(wf, "cuda").eval()


def test_exchanger_matches_reference(golden_dir):
    """exchanger (networks/manipulator.py:18-83), teacher-forced inputs from tests/golden/manipulator.npz: the edited raw and
    both label maps are bit-identical to the reference's (element-wise selection, no arithmetic besides x * 0)."""
    from dmnerf_b200.manipulator import exchanger
    g = dict(np.load(os.path.join(golden_dir, "manipulator.npz")))
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    ori = cu(g["ex_ori_raw"])
    tars = [cu(t) for t in g["ex_tar_raws"]]
    before = _lib.launch_count()
    out, _, lab, tlab = exchanger(ori, tars, cu(g["ex_acc_o"]), [cu(a) for a in g["ex_acc_t"]], [int(v) for v in g["labels"]])
    assert _lib.launch_count() == before + 1
    assert out.data_ptr() == ori.data_ptr()                                   # in place, like the reference
    assert torch.equal(out.cpu(), torch.from_numpy(g["ex_out_raw"]))
    assert torch.equal(lab.cpu(), torch.from_numpy(g["ex_out_label"]))
    assert torch.equal(tlab.cpu(), torch.from_numpy(g["ex_out_tar_label"]))
    assert int((out.cpu() != torch.from_numpy(g["ex_ori_raw"])).any(-1).sum()) > 50       # the case does exchange samples


def _agree(a, b, tol=2e-3):
    """fraction of rays whose map rows agree to `tol` (max over channels)"""
    a = a.detach().cpu().double().numpy() if torch.is_tensor(a) else np.asarray(a, dtype=np.float64)
    b = b.detach().cpu().double().numpy() if torch.is_tensor(b) else np.asarray(b, dtype=np.float64)
    return float((np.abs(a - b).max(-1) <= tol).mean())


def _twin_manipulator(wc, wf, ori, f_tar, S, NI, near, far, labels, us):
    """The oracle edit pipeline carried out in fp64 on the same inputs: how often do the discrete decisions inside
    (arg-max labels, inverse-CDF bins) survive a change of arithmetic at all?"""
    from oracle import dmnerf_oracle as O
    d = torch.float64
    with torch.no_grad():
        return O.manipulator(O.to_torch(wc, d), O.to_torch(wf, d), ori.double(), [t.double() for t in f_tar], S, NI, near, far,
                             labels, us=[u.double() for u in us])


@pytest.mark.parametrize("impl", [_lib.IMPL_SIMT, _lib.IMPL_UMMA])
def test_manipulator_pipeline_matches_reference(golden_dir, impl):
    """manipulator (networks/manipulator.py:137-205): two moved objects, same uniforms as the reference run.  The pipeline
    contains discrete decisions (arg-max labels, importance sampling), so agreement with the reference is measured as the
    fraction of rays whose edited maps match to 2e-3 -- and the yard-stick is the reference's OWN arithmetic in fp64 on the
    same inputs: the native path must agree with the fp32 reference as often as that twin does (40 rays: one ray = 0.025)."""
    from dmnerf_b200.manipulator import manipulator
    from dmnerf_b200.embedder import get_embedder
    g, nc, nf = _manip_setup(golden_dir)
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    labels = [int(v) for v in g["labels"]]
    args = types.SimpleNamespace(N_samples=int(g["n_samples"]), N_importance=int(g["n_importance"]), near=float(g["near"]),
                                 far=float(g["far"]), target_labels=labels)
    us = [cu(u) for u in g["us"]]
    rgb, ins, tar_rgb, tar_acc = manipulator(get_embedder(10)[0], get_embedder(4)[0], nc, nf, cu(g["ori"]), cu(g["f_tar"]), args,
                                             us=us, impl=impl)
    assert rgb.shape == g["final_rgb"].shape and ins.shape == g["final_ins"].shape and tar_acc.shape == g["tar_ins_accum"].shape
    np.testing.assert_allclose(tar_rgb.cpu().numpy(), g["tar_rgb"], rtol=0, atol=2e-4)
    ins_num = int(g["ins_num"])
    wc, wf = synth.make_weights(int(g["seed_c"]), ins_num), synth.make_weights(int(g["seed_f"]), ins_num)
    wc["ins_linear.weight"], wc["ins_linear.bias"] = g["ins_w_c"], g["ins_b_c"]
    wf["ins_linear.weight"], wf["ins_linear.bias"] = g["ins_w_f"], g["ins_b_f"]
    twin = _twin_manipulator(wc, wf, torch.from_numpy(g["ori"]), list(torch.from_numpy(g["f_tar"])), args.N_samples,
                             args.N_importance, args.near, args.far, labels, [torch.from_numpy(u) for u in g["us"]])
    for ours, ref, tw, what in ((rgb, g["final_rgb"], twin[0], "rgb"), (ins, g["final_ins"], twin[1], "ins")):
        r_ours, r_twin = _agree(ours, ref), _agree(tw, ref)
        print("manipulator golden case, %s: ours %.3f, fp64 twin %.3f of rays within 2e-3" % (what, r_ours, r_twin))
        assert r_ours >= r_twin - 0.05, (what, r_ours, r_twin)


@pytest.mark.parametrize("impl", [_lib.IMPL_SIMT, _lib.IMPL_UMMA])
def test_manipulator_pipeline_agreement_at_512_rays(impl):
    """The same comparison on 512 rays (three moved objects), the fp32 oracle (pinned bit for bit to the reference by
    oracle/make_golden_manipulator.py) run live as the reference, its fp64 twin as the yard-stick."""
    from dmnerf_b200.manipulator import manipulator
    from dmnerf_b200.embedder import get_embedder
    from oracle import dmnerf_oracle as O
    ins_num, n, S, NI = 13, 512, 16, 32
    wc, wf = synth.make_weights(31, ins_num), synth.make_weights(32, ins_num)
    rng = np.random.Generator(np.random.PCG64(5))
    for w in (wc, wf):                                   # wide instance heads: every label (and "empty") wins somewhere
        w["ins_linear.weight"] = (w["ins_linear.weight"] * 400).astype(np.float32)
        w["ins_linear.bias"] = (0.3 * rng.standard_normal(ins_num + 1)).astype(np.float32)
    wl = synth.workload("dmsr_study")
    sel = np.linspace(0, 307199, n).astype(np.int64)
    ro, rd = torch.from_numpy(wl["rays_o"][sel]), torch.from_numpy(wl["rays_d"][sel])
    ori = torch.stack([ro, rd], 0)
    tars = []
    for ang, sh in ((0.3, (0.4, -0.2, 0.1)), (-0.2, (-0.3, 0.1, 0.25)), (0.1, (0.1, 0.3, -0.2))):
        c, s_ = float(np.cos(ang)), float(np.sin(ang))
        R = torch.tensor([[c, -s_, 0], [s_, c, 0], [0, 0, 1]], dtype=torch.float32)
        tars.append(torch.stack([ro @ R.T + torch.tensor(sh), rd @ R.T], 0))
    labels = [2, 7, 11]
    gen = torch.Generator().manual_seed(11)
    us = [torch.rand(n, NI, generator=gen) for _ in range(2 + len(tars))]
    near, far = float(wl["near"]), float(wl["far"])
    with torch.no_grad():
        ref = O.manipulator(O.to_torch(wc), O.to_torch(wf), ori, tars, S, NI, near, far, labels, us=us)
    twin = _twin_manipulator(wc, wf, ori, tars, S, NI, near, far, labels, us)
    nc, nf = model_from_weights(wc, "cuda").eval(), model_from_weights(wf, "cuda").eval()
    args = types.SimpleNamespace(N_samples=S, N_importance=NI, near=near, far=far, target_labels=labels)
    before = _lib.launch_count()
    got = manipulator(get_embedder(10)[0], get_embedder(4)[0], nc, nf, ori.cuda(), torch.stack(tars, 0).cuda(), args,
                      us=[u.cuda() for u in us], impl=impl)
    assert _lib.launch_count() - before >= 20
    np.testing.assert_allclose(got[2].cpu().numpy(), ref[2].numpy(), rtol=0, atol=2e-4)      # coarse render of the last target
    for i, what in ((0, "final_rgb"), (1, "final_ins"), (3, "tar_ins_accum")):
        r_ours, r_twin = _agree(got[i], ref[i]), _agree(twin[i], ref[i])
        print("manipulator 512 rays, %s: ours %.3f, fp64 twin %.3f of rays within 2e-3" % (what, r_ours, r_twin))
        assert r_ours >= r_twin - 0.02, (what, r_ours, r_twin)


def test_point_query_matches_embedded_forward():
    """dmnerf_mlp_forward_points (grid sweep of tools/mesh_generator.py:36-49: zero view directions, points embedded in the
    kernel) against the oracle network on the embedded points; a ragged tile included."""
    from dmnerf_b200.autograd import mlp_forward_points
    from dmnerf_b200.testing import model_from_weights, scale_err
    from oracle import dmnerf_oracle as O
    w = synth.make_weights(41, 13)
    net = model_from_weights(w, "cuda").eval()
    gen = torch.Generator().manual_seed(2)
    pts = (torch.rand(1000, 3, generator=gen) * 8 - 4)
    with torch.no_grad():
        got = mlp_forward_points(net, pts.cuda()).cpu().numpy()
        x = torch.cat([O.embed(pts, 10), O.embed(torch.zeros_like(pts), 4)], -1)
        ref = O.mlp_forward(O.to_torch(w), x).numpy()
        vd = torch.randn(1000, 3, generator=gen) * 0.5
        got2 = mlp_forward_points(net, pts.cuda().reshape(10, 100, 3), vd.cuda().reshape(10, 100, 3)).cpu().numpy().reshape(1000, -1)
        ref2 = O.mlp_forward(O.to_torch(w), torch.cat([O.embed(pts, 10), O.embed(vd, 4)], -1)).numpy()
    assert got.shape == (1000, 18)
    assert scale_err(got, ref) <= 1e-4 and scale_err(got2, ref2) <= 1e-4, (scale_err(got, ref), scale_err(got2, ref2))


def test_round2_entry_points_edge_cases():
    """Empty / degenerate inputs of the round-2 entry points: ray selection of zero pixels, a batch with a single object,
    the penalizer on zero rays, the matched loss with every channel matched."""
    import types
    from dmnerf_b200.helpers import get_rays_at
    from dmnerf_b200.evaluator import ins_criterion
    from dmnerf_b200.penalizer import ins_penalizer
    wl = synth.workload("dmsr_study")
    pose = torch.from_numpy(wl["c2w"]).to(DEV)
    ro, rd = get_rays_at(480, 640, wl["K"], pose, torch.zeros(0, dtype=torch.int64))
    assert ro.shape == (0, 3) and rd.shape == (0, 3)
    ro, rd = get_rays_at(480, 640, wl["K"], pose, [0, 307199])
    assert torch.equal(ro[0].cpu(), torch.from_numpy(wl["rays_o"][0])) and torch.equal(rd[1].cpu(), torch.from_numpy(wl["rays_d"][307199]))
    gen = torch.Generator().manual_seed(1)
    pred = torch.sigmoid(torch.randn(33, 5, generator=gen)).to(DEV).requires_grad_(True)
    out = ins_criterion(pred, torch.full((33,), 3.0, device=DEV), 5)              # one object in the batch
    out[0].sum().backward()
    assert torch.isfinite(out[0]).all() and torch.isfinite(pred.grad).all() and float(out[2].sum()) > 0   # 4 unmatched channels
    pred2 = torch.sigmoid(torch.randn(40, 4, generator=gen)).to(DEV)
    lab = (torch.arange(40) % 4).float().to(DEV)
    out2 = ins_criterion(pred2, lab, 4)                                            # every channel matched
    # assignment on the device: the number of distinct labels never reaches the host, invalid_ce is a 0-dim zero
    assert out2[2].shape == () and float(out2[2]) == 0.0 and torch.isfinite(out2[0]).all()
    os.environ["DMNERF_INS_ASSIGN"] = "host"
    try:
        out3 = ins_criterion(pred2, lab, 4)                                        # evaluator.py:33: tensor([0]), shape [1]
    finally:
        del os.environ["DMNERF_INS_ASSIGN"]
    assert out3[2].shape == (1,) and int(out3[2]) == 0 and out3[0].shape == (1,)
    assert abs(float(out3[0]) - float(out2[0])) <= 1e-6 * abs(float(out3[0]))
    args = types.SimpleNamespace(tolerance=0.05, deta_w=0.05)
    loss = ins_penalizer(torch.zeros(0, 64, 18, device=DEV), torch.zeros(0, 64, device=DEV), torch.zeros(0, device=DEV),
                         torch.zeros(0, 3, device=DEV), args)
    assert loss.shape == (1,) and float(loss) == 0.0
