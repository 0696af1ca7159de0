"""GPU: the fp16 preview network (IMPL_UMMA_F16) -- its error against the fp64 oracle and against the fp16 restatement
(oracle/dmnerf_f16.py), reproducibility, independence of the two weight images, re-packing after a weight update, object
selection, manipulation, the fp16 range rule and the training-side rejection.

Bounds against fp64 are the issue's (about 3x over the CPU emulation, tests/test_precision_host.py).  Against the fp16
restatement, the kernel must be much closer than the restatement is to fp64: the two round the same operands to fp16 and
differ only in the fp32 accumulation order (and in the rare activation that lands on the other side of an fp16 rounding
boundary because of it), so FP16_TWIN_FRACTION of the fp16 error is the allowance (measured on an H100: 0.19x at ins_num 13
and 93).  A kernel that dropped or doubled a pass, or rounded anything differently, would sit at 1x or more.  That comparison
uses embedded inputs, which both see bit for bit: in rays mode the kernel forms the points and their sin / cos in fp32, and at
frequency 2^9 that input difference is as large as the fp16 rounding itself (0.3x - 0.6x measured), so rays mode is held to the
fp64 bound only (so is points mode, which embeds fp32 points).  tests/test_gpu_preview_edges.py holds rays and points mode to
the restatement too, run on the kernels' own fp32 inputs (oracle/dmnerf_f16.net_inputs_fp32)."""
import copy
import os
import sys
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from dmnerf_b200 import _lib, synth  # noqa: E402
from oracle import dmnerf_f16 as H  # noqa: E402
from oracle import dmnerf_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F16 = _lib.IMPL_UMMA_F16
NET_REL_L2 = 2e-3
FP16_TWIN_FRACTION = 0.3
RGB_PSNR_DB = 45.0
DEPTH_REL_L2 = 2e-2
LABEL_AGREE = 0.99
MANI_PSNR_DB = 40.0
N_RAYS = 4096


def _workload_case(name):
    from dmnerf_b200.testing import make_models
    wl = synth.workload(name)
    sel = np.linspace(0, wl["H"] * wl["W"] - 1, N_RAYS).astype(np.int64)
    nc, nf, wc, wf = make_models(101, 202, wl["ins_num"], DEV)
    return types.SimpleNamespace(name=name, wl=wl, ro=torch.from_numpy(wl["rays_o"][sel]), rd=torch.from_numpy(wl["rays_d"][sel]),
                                 nc=nc, nf=nf, wc=wc, wf=wf, z=O.z_val_sample(N_RAYS, wl["near"], wl["far"], 64))


_CASES = {}


def _case(name):
    """Models, rays, the fp64 oracle render and the fp16 restatement's render of a workload (built once per module)."""
    if name not in _CASES:
        c = _workload_case(name)
        z64 = O.z_val_sample(N_RAYS, c.wl["near"], c.wl["far"], 64, dtype=torch.float64)
        c.ref = O.render(c.ro.double(), c.rd.double(), O.to_torch(c.wc, torch.float64), O.to_torch(c.wf, torch.float64), z64)
        c.twin = H.render_f16(c.ro, c.rd, O.to_torch(c.wc), O.to_torch(c.wf), z64)
        _CASES[name] = c
    return _CASES[name]


WORKLOADS = ["dmsr_study", "replica_room0_93"]          # ins_num 13 and 93


def _render(c, impl, **kw):
    from dmnerf_b200.render import render_rays
    with torch.no_grad():
        return render_rays(c.ro.to(DEV), c.rd.to(DEV), c.nc, c.nf, c.z[0].to(DEV), want_raw=False, impl=impl, **kw)


def _sync():
    from dmnerf_b200.engine import get_context
    get_context(DEV).sync_check()


@pytest.mark.parametrize("name", WORKLOADS)
def test_network_outputs_against_fp64_and_the_fp16_restatement(name):
    """mlp_forward on embedded inputs, mlp_forward_rays on the oracle's fine depths and mlp_forward_points at the same points
    and view directions: rel. L2 <= 2e-3 against fp64; the embedded call also within FP16_TWIN_FRACTION of the restatement's
    own error against the fp16 restatement."""
    from dmnerf_b200.autograd import mlp_forward, mlp_forward_points, mlp_forward_rays
    c = _case(name)
    n = 512
    ro, rd, zf = c.ro[:n].double(), c.rd[:n].double(), c.ref["z_vals_fine"][:n]
    viewdirs = rd / torch.norm(rd, dim=-1, keepdim=True)
    x, _ = O._net_inputs(ro, rd, viewdirs, zf)
    ref64 = O.mlp_forward(O.to_torch(c.wf, torch.float64), x)
    twin = H.mlp_forward_f16(O.to_torch(c.wf), x)
    with torch.no_grad():
        got_x = mlp_forward(c.nf, x.float().to(DEV), impl=F16).cpu()
        got_r = mlp_forward_rays(c.nf, ro.float().to(DEV), rd.float().to(DEV), zf.float().to(DEV), impl=F16)
        got_r = got_r.reshape(-1, ref64.shape[1]).cpu()
        pts = (ro[:, None, :] + rd[:, None, :] * zf[..., None]).reshape(-1, 3)
        dirs = viewdirs[:, None, :].expand(-1, zf.shape[1], 3).reshape(-1, 3)
        got_p = mlp_forward_points(c.nf, pts.float().to(DEV), dirs.float().to(DEV), impl=F16).cpu()
    _sync()
    e_twin64 = H.rel_l2(twin, ref64)
    for what, got in (("embedded", got_x), ("rays", got_r), ("points", got_p)):
        assert torch.isfinite(got).all(), what
        e64, e16 = H.rel_l2(got, ref64), H.rel_l2(got, twin)
        print("%s %s: rel L2 vs fp64 %.2e (restatement %.2e), vs fp16 restatement %.2e" % (name, what, e64, e_twin64, e16))
        assert e64 <= NET_REL_L2, (what, e64)
        if what == "embedded":
            assert e16 <= FP16_TWIN_FRACTION * e_twin64, (what, e16, e_twin64)


@pytest.mark.parametrize("name", WORKLOADS)
def test_fused_render_against_fp64(name):
    """render_rays (the fused fp16 kernel) on 4096 rays against the fp64 oracle render: arg-max label agreement over all rays;
    rgb PSNR and depth rel. L2 over the rays outside the at most 0.25 % whose importance samples moved to another bin
    (oracle/dmnerf_f16.split_rays: one such ray alone holds the fp16 restatement of dmsr_study to 41.9 dB over all rays).  Every
    ray set aside must be an outlier of the fp16 restatement's own render on the same rays too, so that the exclusion is the
    arithmetic's and cannot hide a kernel fault confined to a few rays."""
    c = _case(name)
    out = _render(c, F16)
    _sync()
    got = {k: v.cpu() for k, v in out.items()}
    typ, outl = H.split_rays(got["rgb_fine"], c.ref["rgb_fine"])
    p = H.psnr(got["rgb_fine"][typ], c.ref["rgb_fine"][typ])
    e_d = H.rel_l2(got["depth_fine"][typ], c.ref["depth_fine"][typ])
    agree = H.label_agreement(got["ins_fine"], c.ref["ins_fine"])
    exact = {k: v.cpu() for k, v in _render(c, _lib.IMPL_UMMA).items()}
    print("%s fp16: rgb PSNR %.1f dB (all rays %.1f; exact kernel %.1f), depth rel L2 %.2e, labels %.4f, %d outlier rays" %
          (name, p, H.psnr(got["rgb_fine"], c.ref["rgb_fine"]), H.psnr(exact["rgb_fine"], c.ref["rgb_fine"]), e_d, agree,
           int(outl.sum())))
    twin_err = (c.twin["rgb_fine"] - c.ref["rgb_fine"]).abs().amax(-1)
    print("%s: rays set aside %s; the restatement's error on them %s" %
          (name, outl.nonzero().flatten().tolist(), [round(float(v), 3) for v in twin_err[outl]]))
    assert bool((twin_err[outl] > 0.05).all()), "a ray set aside is not an outlier of the fp16 restatement"
    assert all(torch.isfinite(v).all() for v in got.values())
    assert p >= RGB_PSNR_DB, p
    assert e_d <= DEPTH_REL_L2, e_d
    assert agree >= LABEL_AGREE, agree


@pytest.mark.parametrize("name", WORKLOADS)
def test_fp16_maps_are_bit_reproducible_and_leave_the_exact_image_alone(name):
    c = _case(name)
    exact_before = _render(c, _lib.IMPL_UMMA)
    a = _render(c, F16)
    b = _render(c, F16)
    exact_after = _render(c, _lib.IMPL_UMMA)
    _sync()
    for k in a:
        assert torch.equal(a[k], b[k]), k
        assert torch.equal(exact_before[k], exact_after[k]), k
    assert not torch.equal(a["rgb_fine"], exact_before["rgb_fine"])          # the two calls did run different networks


def test_in_place_weight_update_repacks_the_fp16_image():
    """An optimizer-style in-place update bumps the parameter versions: the next fp16 call re-packs (the output changes), and
    it equals the output of a fresh model holding the same weights."""
    c = _workload_case("dmsr_study")
    before = _render(c, F16)
    with torch.no_grad():
        c.nf.mlps[3].weight.mul_(1.05)
        c.nc.rgb_feature_linear.weight.add_(0.01)                     # a folded head layer too
    after = _render(c, F16)
    fresh = types.SimpleNamespace(**vars(c))
    fresh.nc, fresh.nf = copy.deepcopy(c.nc), copy.deepcopy(c.nf)
    again = _render(fresh, F16)
    _sync()
    assert not torch.equal(before["rgb_fine"], after["rgb_fine"])
    for k in after:
        assert torch.equal(after[k], again[k]), k


@pytest.mark.parametrize("name", WORKLOADS)
def test_object_selection_at_fp16(name):
    """keep-all gives the unselected fp16 maps bit for bit; keep-{k} and remove-{k} meet the PSNR and label bounds against the
    exact kernel's selected render (PSNR over the typical rays, as in test_fused_render_against_fp64)."""
    c = _case(name)
    ins_num = c.wl["ins_num"]
    plain = _render(c, F16)
    keep_all = _render(c, F16, keep_objects=range(ins_num + 1))
    for k in plain:
        assert torch.equal(plain[k], keep_all[k]), k
    labels = plain["ins_fine"].argmax(-1)
    k_obj = int(torch.mode(labels).values)                              # the object most rays see
    for sel in ([k_obj], [i for i in range(ins_num + 1) if i != k_obj]):
        got = _render(c, F16, keep_objects=sel)
        ref = _render(c, _lib.IMPL_UMMA, keep_objects=sel)
        g_rgb, r_rgb = got["rgb_fine"].cpu(), ref["rgb_fine"].cpu()
        typ, outl = H.split_rays(g_rgb, r_rgb)
        p = H.psnr(g_rgb[typ], r_rgb[typ])
        agree = H.label_agreement(got["ins_fine"].cpu(), ref["ins_fine"].cpu())
        print("%s selection of %d labels: PSNR %.1f dB (all rays %.1f), labels %.4f, %d outlier rays" %
              (name, len(sel), p, H.psnr(g_rgb, r_rgb), agree, int(outl.sum())))
        assert p >= RGB_PSNR_DB and agree >= LABEL_AGREE, (len(sel), p, agree)
    _sync()


def test_manipulate_frame_at_fp16():
    """One edited frame with one moved object: fp16 against exact, same uniforms."""
    from dmnerf_b200.embedder import get_embedder
    from dmnerf_b200.manipulator import manipulate_frame, rigid_rays
    from dmnerf_b200.testing import make_models
    wl = synth.workload("dmsr_study")
    Hh, W = 96, 128
    K = synth.dmsr_intrinsics(Hh, W)
    nc, nf, _, _ = make_models(101, 202, wl["ins_num"], DEV)
    pose = torch.from_numpy(wl["c2w"]).to(DEV)
    move = np.eye(4, dtype=np.float32)
    move[:3, 3] = (0.3, -0.2, 0.1)
    to, td = rigid_rays(Hh, W, K, move, pose)
    args = types.SimpleNamespace(N_test=4096, N_samples=64, N_importance=128, near=wl["near"], far=wl["far"], target_labels=[3],
                                 ins_num=wl["ins_num"])
    pe, ve = get_embedder(10)[0], get_embedder(4)[0]
    maps = {}
    for impl in (_lib.IMPL_UMMA, F16):
        torch.cuda.manual_seed(7)
        maps[impl] = manipulate_frame(Hh, W, K, pose, to[None], td[None], pe, ve, nc, nf, args, impl=impl)
    _sync()
    p = H.psnr(maps[F16][0].cpu(), maps[_lib.IMPL_UMMA][0].cpu())
    print("manipulate_frame fp16 vs exact: PSNR %.1f dB" % p)
    assert torch.isfinite(maps[F16][0]).all()
    assert p >= MANI_PSNR_DB, p


def test_activation_above_fp16_range_is_a_checked_error():
    """A bias that drives the first hidden layer above 65504 (the weights themselves fit): the fp16 call raises and asks for the
    exact path; the exact network still renders the same models afterwards, finite."""
    c = _workload_case("dmsr_study")
    with torch.no_grad():
        c.nc.mlps[0].bias.fill_(1.0e5)
    with pytest.raises(RuntimeError, match="exact"):
        _render(c, F16)
    exact = _render(c, _lib.IMPL_UMMA)
    _sync()
    assert torch.isfinite(exact["rgb_fine"]).all()
    from dmnerf_b200.render import render_frame
    with pytest.raises(RuntimeError, match="exact"):
        render_frame(16, 16, synth.dmsr_intrinsics(16, 16), c.wl["c2w"], c.wl["near"], c.wl["far"], c.nc, c.nf, impl=F16,
                     device=DEV)


def test_range_error_of_both_networks_leaves_no_code_behind():
    """Both networks out of range, on the paths where each network launches on its own (the stage-by-stage path of
    want_raw=True, a sample count other than 64 + 128) and where a batch is rendered in parts (a frame of more than 131 072
    rays).  Each fp16 call raises once; afterwards nothing is pending (sync_check passes) and the exact network renders the
    same models on the same context, finite, on every path."""
    from dmnerf_b200.engine import get_context
    from dmnerf_b200.render import render_frame, render_rays
    c = _workload_case("dmsr_study")
    with torch.no_grad():
        c.nc.mlps[0].bias.fill_(1.0e5)
        c.nf.mlps[0].bias.fill_(1.0e5)
    ctx = get_context(DEV)
    ro, rd = c.ro[:512].to(DEV), c.rd[:512].to(DEV)
    z48 = torch.linspace(c.wl["near"], c.wl["far"], 48, device=DEV)
    frame = lambda impl: render_frame(480, 320, synth.dmsr_intrinsics(480, 320), c.wl["c2w"], c.wl["near"], c.wl["far"], c.nc,
                                      c.nf, impl=impl, device=DEV)
    calls = {"stage path": lambda impl: render_rays(ro, rd, c.nc, c.nf, c.z[0].to(DEV), want_raw=True, impl=impl),
             "48 + 64 samples": lambda impl: render_rays(ro, rd, c.nc, c.nf, z48, N_importance=64, want_raw=False, impl=impl),
             "frame in parts": frame}
    with torch.no_grad():
        for what, call in calls.items():
            with pytest.raises(RuntimeError, match="exact"):
                call(F16)
            ctx.sync_check()
            out = call(_lib.IMPL_UMMA)
            ctx.sync_check()
            key = "rgb" if what == "frame in parts" else "rgb_fine"
            assert torch.isfinite(out[key]).all(), what
        out = render_rays(ro, rd, c.nc, c.nf, c.z[0].to(DEV), want_raw=False, impl=_lib.IMPL_UMMA)
    ctx.sync_check()
    assert torch.isfinite(out["rgb_fine"]).all()


def test_weight_above_fp16_range_fails_at_pack_time():
    c = _workload_case("dmsr_study")
    with torch.no_grad():
        c.nf.mlps[2].weight[0, 0] = 7.0e4
    with pytest.raises(RuntimeError, match="fp16 range"):
        _render(c, F16)
    _render(c, _lib.IMPL_UMMA)
    _sync()


def test_fp16_is_rejected_for_training():
    """IMPL_UMMA_F16 under autograd, and through dmnerf_mlp_forward_train directly, is an error."""
    from dmnerf_b200.autograd import mlp_forward
    from dmnerf_b200.engine import get_context
    from dmnerf_b200.testing import make_models
    nc, _, _, _ = make_models(101, 202, 13, DEV)
    x = torch.rand(256, 90, device=DEV)
    with pytest.raises(RuntimeError, match="inference-only"):
        mlp_forward(nc, x, impl=F16)
    ctx = get_context(DEV)
    ctx.bind(0, nc)
    out = torch.empty(256, 4 + 14, device=DEV)
    acts = torch.empty(256 * ctx.lib.dmnerf_act_floats_per_sample(), device=DEV)
    with pytest.raises(RuntimeError, match="inference-only"):
        ctx.call("dmnerf_mlp_forward_train", ctx.handle, 0, _lib.ptr(x), None, None, None, 256, 1, _lib.ptr(out), _lib.ptr(acts),
                 F16)
