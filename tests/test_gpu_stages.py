"""GPU parity tests, stage by stage with teacher-forced inputs: every CUDA stage kernel is called through
the C ABI (ctypes) and compared with the committed reference fixtures (tests/golden, written from the
unmodified reference) and with the oracle on fresh seeded inputs.

Tolerance (north_star): 1e-4 relative in fp32.  Per-ray quantities use max |err| / max(|ref|, floor) <= 1e-4 with the
floor noted per test.  Network outputs (sums with cancellation) use, per channel group, max |err| / max |ref| <= 1e-4 AND
relL2 <= 1e-4; the exact-fp32 SIMT kernel additionally meets the element-wise bound with a floor of 1% of the scale."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from dmnerf_b200 import synth, _lib
from dmnerf_b200.testing import model_from_weights, max_rel_err, frac_bad, raw_errs

DEV = "cuda"
TOL = 1e-4


def load(golden_dir, name):
    return dict(np.load(os.path.join(golden_dir, name)))


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def test_library_loaded_and_counts_launches():
    lib = _lib.load()
    assert lib.dmnerf_abi_version() == _lib.ABI_VERSION
    assert any("libdmnerf_b200.so" in l for l in open("/proc/self/maps"))


def test_posenc(golden_dir):
    from dmnerf_b200.embedder import get_embedder
    g = load(golden_dir, "embed.npz")
    pe, pd = get_embedder(10)
    ve, vd = get_embedder(4)
    assert (pd, vd) == (63, 27)
    x = cu(g["x"])
    before = _lib.launch_count()
    pos = pe.embed(x).cpu().numpy()
    assert _lib.launch_count() == before + 1
    d = ve.embed(x / x.norm(dim=-1, keepdim=True)).cpu().numpy()
    # |sin|,|cos| <= 1: absolute floor 1e-2 => abs error must stay below 1e-6 on the periodic terms
    assert max_rel_err(pos, g["pos"], 1e-2) <= TOL
    assert max_rel_err(d, g["dir"], 1e-2) <= TOL
    np.testing.assert_array_equal(pos[:, :3], g["x"])
    assert pe.embed(x.reshape(1, -1, 3)).shape == (1, x.shape[0], 63)          # leading dims preserved
    assert pe.embed(x[:0]).shape == (0, 63)                                     # empty input


IMPLS = [pytest.param(_lib.IMPL_SIMT, id="simt"), pytest.param(_lib.IMPL_UMMA, id="umma")]


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("ins_num", [13, 59])
def test_mlp(golden_dir, ins_num, impl):
    """DM_NeRF.forward: fp32 CUDA-core kernel and the wgmma bf16x3 kernel against the reference fixture."""
    from dmnerf_b200.engine import get_context
    g = load(golden_dir, "mlp_ins%d.npz" % ins_num)
    net = model_from_weights(synth.make_weights(int(g["seed"]), ins_num), DEV).eval()
    with torch.no_grad():
        y = net(cu(g["x"]), impl=impl).cpu().numpy()
        get_context(DEV).sync_check()
    assert y.shape == g["y"].shape
    scale = float(np.abs(g["y"]).max())
    e_scale, e_l2 = raw_errs(y, g["y"])
    assert e_scale <= TOL and e_l2 <= TOL, (e_scale, e_l2)
    if impl == _lib.IMPL_SIMT:
        assert max_rel_err(y, g["y"], 1e-2 * scale) <= TOL
    # element-wise view of the same comparison (DESIGN section 2: the scale-relative metric above is a relaxation of "1e-4 rel"):
    # fraction of outputs with |err| <= 1e-4 * max(|ref|, 0.1 * scale of their channel group)
    within = []
    for sl in (slice(0, 3), slice(3, 4), slice(4, None)):
        ref_g, got_g = g["y"][..., sl].astype(np.float64), y[..., sl].astype(np.float64)
        gs = float(np.abs(ref_g).max())
        within.append((np.abs(got_g - ref_g) <= 1e-4 * np.maximum(np.abs(ref_g), 0.1 * gs)).mean())
    print("test_mlp ins %d impl %d: fraction of outputs within 1e-4 element-wise (rgb, sigma, ins) = %s" % (ins_num, impl, within))
    assert min(within) >= 0.995, within
    with torch.no_grad():                                                      # ragged: 1 row, 65 rows, 0 rows
        for m in (1, 65, 0):
            ym = net(cu(g["x"][:m]), impl=impl).cpu().numpy()
            assert ym.shape == (m, 4 + ins_num + 1)
            if m:
                assert max(raw_errs(ym, g["y"][:m])) <= TOL


def test_composite(golden_dir):
    from dmnerf_b200.render import composite, render_train
    g = load(golden_dir, "composite.npz")
    with torch.no_grad():
        rgb, w, depth, ins, acc = composite(cu(g["raw"]), cu(g["z"]), cu(g["rays_d"]))
        r4 = render_train(cu(g["raw"]), cu(g["z"]), cu(g["rays_d"]))
    assert len(r4) == 4 and r4[3].shape == g["ins"].shape
    assert max_rel_err(w.cpu(), g["weights"], 1e-3) <= TOL
    assert max_rel_err(rgb.cpu(), g["rgb"], 1e-2) <= TOL
    assert max_rel_err(depth.cpu(), g["depth"], 1e-1) <= TOL
    assert max_rel_err(ins.cpu(), g["ins"], 1e-2) <= TOL
    assert max_rel_err(acc.cpu(), g["weights"].sum(-1), 1e-2) <= TOL
    assert float(w[0].abs().max()) == 0.0 and float(acc.max()) <= 1.0 + 1e-5
    # manipulator_render variant keeps all ins_num+1 channels (manipulator.py:86-105)
    with torch.no_grad():
        ins_all = composite(cu(g["raw"]), cu(g["z"]), cu(g["rays_d"]), keep_all_ins=True)[3]
    assert ins_all.shape[1] == g["ins"].shape[1] + 1
    np.testing.assert_allclose(ins_all[:, :-1].cpu().numpy(), ins.cpu().numpy(), rtol=0, atol=0)


def test_sample_pdf_and_sort(golden_dir):
    from dmnerf_b200.helpers import sample_pdf, sort_concat
    g = load(golden_dir, "sample_pdf.npz")
    b, w = cu(g["bins"]), cu(g["weights"])
    det = sample_pdf(b, w, 128, det=True).cpu().numpy()
    rnd = sample_pdf(b, w, 128, det=False, u=cu(g["u"])).cpu().numpy()
    # the inverse CDF is discontinuous where a bin's mass is below 1e-5 (helpers.py:151): allow a handful of
    # samples to land on the other side of such a jump, everything else must match to 1e-4 relative
    for got, ref in ((det, g["det"]), (rnd, g["rnd"])):
        assert frac_bad(got, ref, TOL, 1e-5) <= 2e-3
        assert np.isfinite(got).all() and got.min() >= g["bins"].min() - 1e-4 and got.max() <= g["bins"].max() + 1e-4
    assert (np.diff(det, axis=-1) >= -1e-6).all()                               # det sampling is monotone
    a = cu(np.sort(g["bins"], -1))
    merged = sort_concat(a, cu(g["rnd"])).cpu().numpy()
    np.testing.assert_array_equal(merged, np.sort(np.concatenate([g["bins"], g["rnd"]], -1), -1))
    dup = cu(np.array([[3., 1., 1., 2.]], dtype=np.float32))                     # ties
    np.testing.assert_array_equal(sort_concat(dup, dup).cpu().numpy(), [[1, 1, 1, 1, 2, 2, 3, 3]])


def _render_inputs(golden_dir, tag):
    g = load(golden_dir, "render_%s.npz" % tag)
    ins_num = int(g["ins_num"])
    nc = model_from_weights(synth.make_weights(int(g["seed_coarse"]), ins_num), DEV).eval()
    nf = model_from_weights(synth.make_weights(int(g["seed_fine"]), ins_num), DEV).eval()
    return g, nc, nf, ins_num


@pytest.mark.parametrize("tag", ["study", "room0"])
@pytest.mark.parametrize("impl", IMPLS)
def test_render_stagewise_vs_reference(golden_dir, tag, impl):
    """dm_nerf() through the drop-in API against the reference's fixture, stage-wise with teacher forcing:
    each stage is fed the REFERENCE's intermediate so the sample_pdf amplification (SURVEY 7) is not compounded."""
    import types
    from dmnerf_b200.render import dm_nerf, composite
    from dmnerf_b200.embedder import get_embedder
    from dmnerf_b200.helpers import z_val_sample
    from dmnerf_b200.autograd import mlp_forward_rays
    from dmnerf_b200.helpers import sample_pdf, sort_concat
    g, nc, nf, ins_num = _render_inputs(golden_dir, tag)
    ro, rd = cu(g["rays_o"]), cu(g["rays_d"])
    n = ro.shape[0]
    with torch.no_grad():
        # stage 1: coarse network on the reference's coarse depths
        raw_c = mlp_forward_rays(nc, ro, rd, cu(g["det_z_vals_coarse"]), impl).cpu().numpy()
        assert max(raw_errs(raw_c, g["det_raw_coarse"])) <= TOL
        # stage 2: composite of the reference's raw
        rgb, w, depth, ins, acc = composite(cu(g["det_raw_coarse"]), cu(g["det_z_vals_coarse"]), rd)
        assert max_rel_err(rgb.cpu(), g["det_rgb_coarse"], 1e-2) <= TOL
        assert max_rel_err(depth.cpu(), g["det_depth_coarse"], 1e-1) <= TOL
        assert max_rel_err(ins.cpu(), g["det_ins_coarse"], 1e-2) <= TOL
        # stage 3: fine network on the reference's fine depths, composite of the reference's raw
        raw_f = mlp_forward_rays(nf, ro, rd, cu(g["det_z_vals_fine"]), impl).cpu().numpy()
        assert max(raw_errs(raw_f, g["det_raw_fine"])) <= TOL
        rgb, w, depth, ins, acc = composite(cu(g["det_raw_fine"]), cu(g["det_z_vals_fine"]), rd)
        assert max_rel_err(rgb.cpu(), g["det_rgb_fine"], 1e-2) <= TOL
        assert max_rel_err(depth.cpu(), g["det_depth_fine"], 1e-1) <= TOL
        assert max_rel_err(ins.cpu(), g["det_ins_fine"], 1e-2) <= TOL

        # end to end through the reference call surface (ill-conditioned by construction: looser bound)
        args = types.SimpleNamespace(perturb=0.0, N_importance=128, is_train=False, N_ins=None)
        pe, _ = get_embedder(10)
        ve, _ = get_embedder(4)
        zc = z_val_sample(n, float(g["near"]), float(g["far"]), 64, device=DEV)
        assert zc.stride(0) == 0
        out = dm_nerf(torch.stack([ro, rd], 0), pe, ve, nc, nf, zc, args)
        # yard-stick for the ill-conditioned end-to-end comparison: how far the reference's own arithmetic moves when
        # it is carried out in fp64 instead of fp32 (SURVEY.md section 7)
        from oracle import dmnerf_oracle as O
        wc, wf = synth.make_weights(int(g["seed_coarse"]), ins_num), synth.make_weights(int(g["seed_fine"]), ins_num)
        twin = O.render(ro.cpu().double(), rd.cpu().double(), O.to_torch(wc, torch.float64), O.to_torch(wf, torch.float64),
                        O.z_val_sample(n, float(g["near"]), float(g["far"]), 64, dtype=torch.float64))
    for k in ("rgb_fine", "ins_fine", "z_vals_fine", "raw_fine", "raw_coarse", "rgb_coarse", "ins_coarse",
              "z_vals_coarse", "depth_fine", "depth_coarse"):
        assert k in out and tuple(out[k].shape) == g["det_" + k].shape, k
        assert np.isfinite(out[k].cpu().numpy()).all()
    np.testing.assert_allclose(out["z_vals_coarse"].cpu().numpy(), g["det_z_vals_coarse"], rtol=0, atol=0)
    np.testing.assert_allclose(out["rgb_coarse"].cpu().numpy(), g["det_rgb_coarse"], rtol=1e-4, atol=1e-5)
    for k, floor in (("z_vals_fine", 1e-3), ("rgb_fine", 1e-4), ("depth_fine", 1e-3), ("ins_fine", 1e-4)):
        ref = g["det_" + k]
        dev_twin = float(np.abs(twin[k].float().numpy() - ref).max())
        dev_ours = float(np.abs(out[k].cpu().numpy() - ref).max())
        assert dev_ours <= 10.0 * dev_twin + floor, (k, dev_ours, dev_twin)
    z = out["z_vals_fine"]
    assert bool((z[:, 1:] >= z[:, :-1]).all())


@pytest.mark.parametrize("impl", IMPLS)
def test_render_perturb_uses_given_uniforms(golden_dir, impl):
    from dmnerf_b200.render import render_rays
    g, nc, nf, ins_num = _render_inputs(golden_dir, "study")
    ro, rd = cu(g["rays_o"]), cu(g["rays_d"])
    zc = cu(np.broadcast_to(g["det_z_vals_coarse"][:1], g["det_z_vals_coarse"].shape).copy())
    with torch.no_grad():
        out = render_rays(ro, rd, nc, nf, zc, perturb=1.0, N_importance=128, t_rand=cu(g["t_rand"]), u=cu(g["u"]), impl=impl)
    np.testing.assert_allclose(out["z_vals_coarse"].cpu().numpy(), g["trn_z_vals_coarse"], rtol=0, atol=2e-6)
    assert max(raw_errs(out["raw_coarse"].cpu().numpy(), g["trn_raw_coarse"])) <= TOL
    np.testing.assert_allclose(out["rgb_coarse"].cpu().numpy(), g["trn_rgb_coarse"], rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(out["rgb_fine"].cpu().numpy(), g["trn_rgb_fine"], rtol=0, atol=5e-3)


def test_full_frame_properties_and_chunk_invariance():
    """BASELINE config 2 size (640x480, 64+128): properties that do not need the oracle."""
    from dmnerf_b200.render import render_rays
    from dmnerf_b200.testing import make_models
    wl = synth.workload("dmsr_study")
    nc, nf, _, _ = make_models(101, 202, wl["ins_num"], DEV)
    ro, rd = cu(wl["rays_o"]), cu(wl["rays_d"])
    z = torch.linspace(0, 1, 64, device=DEV) * (wl["far"] - wl["near"]) + wl["near"]
    n = 40960                                                                    # 10 reference chunks (N_test=4096)
    with torch.no_grad():
        full = render_rays(ro[:n], rd[:n], nc, nf, z, want_raw=False, want_samples=True)
        part = render_rays(ro[4096:8192], rd[4096:8192], nc, nf, z, want_raw=False, want_samples=True)
    zf = full["z_vals_fine"]
    assert bool((zf[:, 1:] >= zf[:, :-1]).all())
    assert float(zf.min()) >= wl["near"] - 1e-4 and float(zf.max()) <= wl["far"] + 1e-4
    assert float(full["acc_fine"].max()) <= 1.0 + 1e-4 and float(full["acc_fine"].min()) >= 0.0
    assert float(full["acc_fine"].mean()) > 0.5                                   # trained-like weights terminate rays
    assert bool(((full["ins_fine"] > 0) & (full["ins_fine"] < 1)).all())
    for k in ("rgb_fine", "depth_fine", "ins_fine", "z_vals_fine", "rgb_coarse"):
        assert torch.isfinite(full[k]).all()
        assert torch.equal(full[k][4096:8192], part[k]), k                       # rays are independent units


@pytest.mark.parametrize("n_rays,perturb", [(1001, 0.0), (258, 1.0), (1, 0.0)])
def test_fused_render_matches_unfused(n_rays, perturb):
    """The single-kernel pipeline (coarse net -> composite -> sampling -> fine net -> composite, nothing per-sample in HBM)
    against the stage-by-stage kernels fed by the same tensor-core network: same depths, same maps; odd ray counts
    exercise the half-empty last ray pair."""
    from dmnerf_b200.render import render_rays
    from dmnerf_b200.engine import get_context
    from dmnerf_b200.testing import make_models
    wl = synth.workload("replica_room0")
    nc, nf, _, _ = make_models(11, 12, wl["ins_num"], DEV)
    sel = np.linspace(0, 307199, n_rays).astype(np.int64)
    ro, rd = cu(wl["rays_o"][sel]), cu(wl["rays_d"][sel])
    z = torch.linspace(0, 1, 64, device=DEV) * (wl["far"] - wl["near"]) + wl["near"]
    gen = torch.Generator(device=DEV).manual_seed(9)
    kw = {}
    if perturb:
        kw = dict(t_rand=torch.rand((n_rays, 64), device=DEV, generator=gen), u=torch.rand((n_rays, 128), device=DEV, generator=gen))
    with torch.no_grad():
        get_context(DEV).bind(0, nc); get_context(DEV).bind(1, nf)                # weight packing launches happen here
        before = _lib.launch_count()
        fused = render_rays(ro, rd, nc, nf, z, perturb=perturb, want_raw=False, want_samples=True, impl=_lib.IMPL_UMMA, **kw)
        assert _lib.launch_count() - before == 1                                   # ONE kernel for the whole pipeline
        ref = render_rays(ro, rd, nc, nf, z, perturb=perturb, want_raw=True, impl=_lib.IMPL_UMMA, **kw)
        get_context(DEV).sync_check()
    np.testing.assert_allclose(fused["z_vals_coarse"].cpu().numpy(), ref["z_vals_coarse"].cpu().numpy(), rtol=0, atol=0)
    for k, tol in (("rgb_coarse", 2e-6), ("depth_coarse", 2e-5), ("acc_coarse", 2e-6), ("ins_coarse", 2e-6), ("weights_coarse", 2e-6)):
        np.testing.assert_allclose(fused[k].cpu().numpy(), ref[k].cpu().numpy(), rtol=1e-5, atol=tol, err_msg=k)
    # the fine depths come from the coarse weights: tiny differences may flip a sample across a pdf jump in isolated rays
    zf_f, zf_r = fused["z_vals_fine"].cpu().numpy(), ref["z_vals_fine"].cpu().numpy()
    same = np.abs(zf_f - zf_r).max(-1) <= 1e-5
    assert same.mean() >= 0.98
    for k, tol in (("rgb_fine", 5e-6), ("depth_fine", 5e-5), ("acc_fine", 5e-6), ("ins_fine", 5e-6), ("weights_fine", 5e-6)):
        np.testing.assert_allclose(fused[k].cpu().numpy()[same], ref[k].cpu().numpy()[same], rtol=1e-4, atol=tol, err_msg=k)
    assert all(torch.isfinite(v).all() for v in fused.values())


def test_errors_are_loud():
    from dmnerf_b200.render import render_rays
    from dmnerf_b200.testing import make_models
    with pytest.raises(RuntimeError):
        render_rays(torch.zeros(4, 3), torch.zeros(4, 3), None, None, torch.zeros(64))   # CPU tensors
    lib = _lib.load()
    rc = lib.dmnerf_posenc(None, 5, 10, None, None)
    assert rc != 0 and b"NULL" in lib.dmnerf_last_error()


@pytest.mark.parametrize("impl", IMPLS)
def test_baseline_config1_coarse_only_1024_rays(impl):
    """BASELINE configs[0]: DM-SR 'study', 1024-ray chunk, 64 coarse samples, coarse MLP only -- against the oracle run
    on the host (the reference's CPU-runnable case)."""
    from dmnerf_b200.render import composite
    from dmnerf_b200.autograd import mlp_forward_rays
    from dmnerf_b200.testing import make_models
    from oracle import dmnerf_oracle as O
    wl = synth.workload("dmsr_study")
    nc, _, wc, _ = make_models(101, 202, 13, DEV)
    ro, rd = torch.from_numpy(wl["rays_o"][:1024]), torch.from_numpy(wl["rays_d"][:1024])
    z = O.z_val_sample(1024, wl["near"], wl["far"], 64)
    with torch.no_grad():
        x, shp = O._net_inputs(ro, rd, rd / rd.norm(dim=-1, keepdim=True), z)
        raw_ref = O.mlp_forward(O.to_torch(wc), x).reshape(1024, 64, -1)
        rgb_ref, w_ref, d_ref, ins_ref, acc_ref = O.composite(raw_ref, z, rd)
        raw = mlp_forward_rays(nc, ro.to(DEV), rd.to(DEV), z.contiguous().to(DEV), impl)
        rgb, w, depth, ins, acc = composite(raw, z.contiguous().to(DEV), rd.to(DEV))
    assert max(raw_errs(raw.cpu().numpy(), raw_ref.numpy())) <= TOL
    assert max_rel_err(rgb.cpu(), rgb_ref, 1e-2) <= TOL
    assert max_rel_err(depth.cpu(), d_ref, 1e-1) <= TOL
    assert max_rel_err(ins.cpu(), ins_ref, 1e-2) <= TOL
    assert float((w.cpu() - w_ref).abs().max()) <= TOL          # weights live in [0, 1]


@pytest.mark.parametrize("name", ["replica_room0", "replica_room0_93", "replica_office2"])
def test_baseline_replica_configs_full_width_object_head(name):
    """BASELINE configs[2] / [4] shapes: Replica intrinsics, near 0, 59 / 93 / 69 objects (C = 64 / 98 / 74 channels): the
    fused render against the stage-by-stage path on 2048 rays, plus range properties."""
    from dmnerf_b200.render import render_rays
    from dmnerf_b200.testing import make_models
    wl = synth.workload(name)
    ins = wl["ins_num"]
    nc, nf, _, _ = make_models(31, 32, ins, DEV)
    sel = np.linspace(0, 307199, 2048).astype(np.int64)
    ro, rd = cu(wl["rays_o"][sel]), cu(wl["rays_d"][sel])
    z = torch.linspace(0, 1, 64, device=DEV) * (wl["far"] - wl["near"]) + wl["near"]
    with torch.no_grad():
        fused = render_rays(ro, rd, nc, nf, z, want_raw=False, want_samples=True)
        ref = render_rays(ro, rd, nc, nf, z, want_raw=True)
    assert fused["ins_fine"].shape == (2048, ins) and ref["raw_fine"].shape == (2048, 192, 4 + ins + 1)
    same = (fused["z_vals_fine"] - ref["z_vals_fine"]).abs().amax(-1) <= 1e-5
    assert float(same.float().mean()) >= 0.98
    for k in ("rgb_fine", "ins_fine", "depth_fine", "acc_fine", "rgb_coarse", "ins_coarse"):
        a, b = fused[k][same] if k.endswith("fine") else fused[k], ref[k][same] if k.endswith("fine") else ref[k]
        assert torch.isfinite(a).all()
        np.testing.assert_allclose(a.cpu().numpy(), b.cpu().numpy(), rtol=1e-4, atol=5e-5, err_msg=k)
    assert bool(((fused["ins_fine"] > 0) & (fused["ins_fine"] < 1)).all())
    assert float(fused["acc_fine"].max()) <= 1.0 + 1e-4


def test_get_rays_k_kernel_matches_reference(golden_dir):
    """SURVEY 8(f1): ray generation (networks/helpers.py:50-61) as a kernel, against the reference's own rays."""
    from dmnerf_b200.helpers import get_rays_k
    g = load(golden_dir, "rays.npz")
    o, d = get_rays_k(480, 640, g["K"], cu(g["c2w"]))
    assert o.shape == (480, 640, 3) and d.shape == (480, 640, 3)
    np.testing.assert_allclose(d.reshape(-1, 3)[g["idx"]].cpu().numpy(), g["rays_d"], rtol=1e-6, atol=1e-7)
    np.testing.assert_array_equal(o.reshape(-1, 3)[g["idx"]].cpu().numpy(), g["rays_o"])
    wl = synth.workload("replica_room0")
    o2, d2 = get_rays_k(wl["H"], wl["W"], wl["K"], cu(wl["c2w"]))
    np.testing.assert_allclose(d2.reshape(-1, 3).cpu().numpy(), wl["rays_d"], rtol=1e-6, atol=1e-7)
