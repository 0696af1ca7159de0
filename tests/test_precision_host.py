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
