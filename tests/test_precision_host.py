"""CPU checks of the fp16 preview network (DMNERF_IMPL_UMMA_F16): the fp16 oracle's error against fp64 on the workloads (the
origin of the GPU bounds in test_gpu_precision.py), the shipped library's fp16 kernels, and which calls DMNERF_INFER_IMPL
reaches."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from dmnerf_b200 import synth  # noqa: E402
from oracle import dmnerf_f16 as H  # noqa: E402
from oracle import dmnerf_oracle as O  # noqa: E402

# The GPU bounds (test_gpu_precision.py); the fp16 oracle must meet them with margin on the same kind of rays.
NET_REL_L2 = 2e-3
RGB_PSNR_DB = 45.0
DEPTH_REL_L2 = 2e-2
LABEL_AGREE = 0.99


def _case(name, n_rays):
    wl = synth.workload(name)
    sel = np.linspace(0, wl["H"] * wl["W"] - 1, n_rays).astype(np.int64)
    ro = torch.from_numpy(wl["rays_o"][sel]).double()
    rd = torch.from_numpy(wl["rays_d"][sel]).double()
    wc = synth.make_weights(101, wl["ins_num"])
    wf = synth.make_weights(202, wl["ins_num"])
    z = O.z_val_sample(n_rays, wl["near"], wl["far"], 64, dtype=torch.float64)
    return ro, rd, wc, wf, z


@pytest.mark.parametrize("name,n_rays", [("dmsr_study", 384), ("replica_room0_93", 256)])
def test_fp16_oracle_meets_the_gpu_bounds_against_fp64(name, n_rays):
    ro, rd, wc, wf, z = _case(name, n_rays)
    p64c, p64f = O.to_torch(wc, torch.float64), O.to_torch(wf, torch.float64)
    ref = O.render(ro, rd, p64c, p64f, z)
    # network, teacher-forced on the fp64 render's fine depths
    viewdirs = rd / torch.norm(rd, dim=-1, keepdim=True)
    x, _ = O._net_inputs(ro, rd, viewdirs, ref["z_vals_fine"])
    net64 = O.mlp_forward(p64f, x)
    net16 = H.mlp_forward_f16(O.to_torch(wf), x)
    e_net = H.rel_l2(net16, net64)
    # end to end, through sample_pdf
    got = H.render_f16(ro, rd, O.to_torch(wc), O.to_torch(wf), z)
    typ, out = H.split_rays(got["rgb_fine"], ref["rgb_fine"])
    p = H.psnr(got["rgb_fine"][typ], ref["rgb_fine"][typ])
    e_depth = H.rel_l2(got["depth_fine"][typ], ref["depth_fine"][typ])
    agree = H.label_agreement(got["ins_fine"], ref["ins_fine"])
    print("%s: net rel L2 %.2e, rgb PSNR %.1f dB (all rays %.1f), depth rel L2 %.2e, labels %.4f, %d outlier rays" %
          (name, e_net, p, H.psnr(got["rgb_fine"], ref["rgb_fine"]), e_depth, agree, int(out.sum())))
    assert e_net <= NET_REL_L2 / 3, e_net
    assert p >= RGB_PSNR_DB + 5.0, p
    assert e_depth <= DEPTH_REL_L2 / 2, e_depth
    assert agree >= LABEL_AGREE, agree


def test_fp16_oracle_rounds_its_operands():
    """The restatement is not the exact network in disguise: its error against fp64 is orders above the fp32 network's."""
    ro, rd, wc, wf, z = _case("dmsr_study", 32)
    viewdirs = rd / torch.norm(rd, dim=-1, keepdim=True)
    x, _ = O._net_inputs(ro, rd, viewdirs, z)
    net64 = O.mlp_forward(O.to_torch(wc, torch.float64), x)
    e32 = H.rel_l2(O.mlp_forward(O.to_torch(wc), x.float()), net64)
    e16 = H.rel_l2(H.mlp_forward_f16(O.to_torch(wc), x), net64)
    assert e16 > 30 * e32, (e16, e32)


@pytest.mark.parametrize("name", ["dmsr_study", "replica_room0_93"])
def test_fp32_twin_inputs_are_within_a_few_ulp_of_the_fp64_embedding(name):
    """net_inputs_fp32 and points_inputs_fp32 (the kernels' fp32 inputs) against O.embed of the same rays in fp64: every column
    within 4 fp32 ulp (2^-23) of (2^k |x| + 1), where 2^k is the column's frequency and |x| the scale of its coordinate
    (|o| + |d z| for a point, |viewdir| for a direction).  The identity columns are the fp32 point and direction themselves."""
    ro, rd, _, _, _ = _case(name, 48)
    ro, rd = ro.float(), rd.float()
    gen = torch.Generator().manual_seed(3)
    wl = synth.workload(name)
    z = (torch.rand(48, 37, generator=gen, dtype=torch.float64) * (wl["far"] - wl["near"]) + wl["near"]).float()
    twin = H.net_inputs_fp32(ro, rd, z).double()
    ro64, rd64, z64 = ro.double(), rd.double(), z.double()
    vd64 = rd64 / torch.norm(rd64, dim=-1, keepdim=True)
    x64, _ = O._net_inputs(ro64, rd64, vd64, z64)
    pt_scale = (ro64.abs()[:, None, :] + (rd64[:, None, :] * z64[..., None]).abs()).reshape(-1, 3)
    vd_scale = vd64.abs()[:, None, :].expand(48, 37, 3).reshape(-1, 3)
    ulp = 2.0 ** -23
    tol = torch.cat([4 * ulp * (H.embed_freq_scale(10) * pt_scale.repeat(1, 21) + 1),
                     4 * ulp * (H.embed_freq_scale(4) * vd_scale.repeat(1, 9) + 1)], -1)
    err = (twin - x64).abs()
    assert bool((err <= tol).all()), float((err / tol).max())
    assert float(err[:, 3 + 6 * 9:63].max()) > 0.0           # the fp32 inputs are not fp64 in disguise
    # points mode: the fp32 points and directions embedded as they are
    pts = (ro[:, None, :] + rd[:, None, :] * z[..., None]).reshape(-1, 3)
    dirs = (rd / torch.norm(rd, dim=-1, keepdim=True))[:, None, :].expand(48, 37, 3).reshape(-1, 3)
    xp = H.points_inputs_fp32(pts, dirs).double()
    xp64 = torch.cat([O.embed(pts.double(), 10), O.embed(dirs.double(), 4)], -1)
    assert torch.equal(xp[:, :3], pts.double()) and torch.equal(xp[:, 63:66], dirs.double())
    assert float((xp - xp64).abs().max()) <= 2 * ulp


@pytest.mark.parametrize("keep_all_ins", [False, True])
def test_render_on_depths_reproduces_the_oracle_render(keep_all_ins):
    """render_on_depths with the fp64 network and fp64 inputs, on O.render's own coarse and fine depths, gives O.render's maps
    and weights to fp64 rounding; with an object selection, objects_oracle.render's.  Labels are the first maximum of the
    instance sigmoids and the gap is the distance to the second largest."""
    from oracle import objects_oracle as OO
    ro, rd, wc, wf, z = _case("dmsr_study", 40)
    p64c, p64f = O.to_torch(wc, torch.float64), O.to_torch(wf, torch.float64)
    net_c, net_f = (lambda x: O.mlp_forward(p64c, x)), (lambda x: O.mlp_forward(p64f, x))
    ins_num = wc["ins_linear.weight"].shape[0] - 1
    keep = torch.zeros(ins_num + 1, dtype=torch.bool)
    keep[[0, 2, 5, ins_num]] = True
    for sel in (None, keep):
        ref = O.render(ro, rd, p64c, p64f, z) if sel is None else OO.render(ro, rd, p64c, p64f, z, sel)
        got = H.render_on_depths(net_c, net_f, ro, rd, ref["z_vals_coarse"], ref["z_vals_fine"], fp32_inputs=False, keep=sel,
                                 keep_all_ins=keep_all_ins)
        for p in ("coarse", "fine"):
            want = O.composite(ref["raw_" + p] if sel is None else OO.select_objects(ref["raw_" + p], sel), ref["z_vals_" + p],
                               rd, keep_all_ins=keep_all_ins)
            for k, v in zip(("rgb", "weights", "depth", "ins", "acc"), want):
                assert torch.allclose(got["%s_%s" % (k, p)], v, rtol=1e-12, atol=1e-12), (k, p)
            if not keep_all_ins:
                for k in ("rgb", "depth", "ins", "acc", "weights"):
                    assert torch.allclose(got["%s_%s" % (k, p)], ref["%s_%s" % (k, p)], rtol=1e-12, atol=1e-12), (k, p)
            raw = got["raw_" + p]
            assert torch.allclose(raw, ref["raw_" + p], rtol=1e-12, atol=1e-12)
            assert torch.equal(got["labels_" + p], OO.object_labels(raw))
            s = torch.sigmoid(raw[..., 4:]).sort(-1, descending=True).values
            assert torch.equal(got["gap_" + p], s[..., 0] - s[..., 1]) and bool((got["gap_" + p] >= 0).all())


def _sass_counts():
    path = os.path.join(ROOT, "dm-nerf_b200", "lib", "libdmnerf_b200.so")
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    if not os.path.exists(path):
        pytest.skip("library not built")
    out = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    per, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = per.setdefault(m.group(1), {"HGMMA_F16": 0, "HGMMA_BF16": 0, "UBLKCP": 0})
            continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)(\.\S+)?", line)
        if m and cur is not None:
            op, mods = m.group(1), m.group(2) or ""
            if op == "HGMMA":
                cur["HGMMA_BF16" if ".BF16" in mods else "HGMMA_F16"] += 1
            elif op == "UBLKCP":
                cur["UBLKCP"] += 1
    return per


def test_fp16_kernels_issue_fp16_hgmma_and_fewer_than_their_exact_twins():
    """cuobjdump -sass of the built library: each fp16 instantiation issues HGMMA with fp16 operands only, streams its weights
    with UBLKCP, and has fewer HGMMA instructions than the exact kernel it mirrors."""
    per = _sass_counts()
    twins = {"mlp_f16_kernelILb0E": "mlp_umma_kernelILb0E", "mlp_f16_kernelILb1E": "mlp_umma_kernelILb1E",
             "render_objects_f16_kernel": "render_objects_kernel"}
    for f16, exact in twins.items():
        fk = [c for k, c in per.items() if f16 in k]
        ek = [c for k, c in per.items() if exact in k and "f16" not in k]
        assert len(fk) == 1 and len(ek) == 1, (f16, len(fk), len(ek))
        f, e = fk[0], ek[0]
        assert f["HGMMA_F16"] > 0 and f["HGMMA_BF16"] == 0, (f16, f)
        assert e["HGMMA_BF16"] > 0 and e["HGMMA_F16"] == 0, (exact, e)
        assert f["UBLKCP"] > 0, (f16, f)
        assert f["HGMMA_F16"] < e["HGMMA_BF16"], (f16, f, e)


_PROBE = """
import sys
sys.path.insert(0, %r)
from dmnerf_b200 import _lib, backward
print(_lib.infer_impl(_lib.IMPL_AUTO), _lib.infer_impl(_lib.IMPL_UMMA), _lib.infer_impl(_lib.IMPL_SIMT),
      backward._train_impl(_lib.IMPL_AUTO))
try:
    backward._train_impl(_lib.IMPL_UMMA_F16)
    print("accepted")
except RuntimeError:
    print("rejected")
""" % ROOT


@pytest.mark.parametrize("env,auto", [("f16", 3), ("F16", 3), ("", 0), ("exact", 0)])
def test_infer_impl_switch_resolves_only_inference_calls(env, auto):
    """DMNERF_INFER_IMPL=f16 turns IMPL_AUTO of inference calls into IMPL_UMMA_F16; explicit choices stay; the training forward
    resolves IMPL_AUTO to its exact network whatever the switch says, and rejects IMPL_UMMA_F16."""
    env_vars = dict(os.environ, DMNERF_INFER_IMPL=env)
    out = subprocess.run([sys.executable, "-c", _PROBE], capture_output=True, text=True, env=env_vars, check=True).stdout.split()
    assert out[:3] == [str(auto), "2", "1"], out
    assert out[3] in ("1", "2"), out                     # IMPL_UMMA (default) or IMPL_SIMT (DMNERF_TRAIN_IMPL=simt)
    assert out[4] == "rejected", out


def test_inference_entry_points_resolve_the_switch():
    """Every inference entry point that takes impl resolves it through _lib.infer_impl (and only _lib reads the variable)."""
    pkg = os.path.join(ROOT, "dm-nerf_b200")
    for mod, funcs in {"render.py": ("render_rays", "render_frame"),
                       "autograd.py": ("mlp_forward", "mlp_forward_rays", "mlp_forward_points")}.items():
        src = open(os.path.join(pkg, mod)).read()
        for fn in funcs:
            body = re.search(r"\ndef %s\(.*?(?=\ndef |\nclass |\Z)" % fn, src, re.S).group(0)
            assert "_lib.infer_impl(impl)" in body, (mod, fn)
    readers = [f for f in os.listdir(pkg) if f.endswith(".py") and "DMNERF_INFER_IMPL\"" in open(os.path.join(pkg, f)).read()]
    assert readers == ["_lib.py"], readers
