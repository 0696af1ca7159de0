"""Where the time of the reference's whole training iteration (train_dmsr.py:23-64 through the drop-in call surface) goes:
event-timed iteration, GPU-busy time (sum of kernel durations from CUPTI), host-issue time (the same loop with the GPU idle at
the start of every iteration cannot run faster than the host can issue it), top kernels.  python tools/prof_full_iter.py"""
import os
import time
import types

import numpy as np
import torch

from _harness import cuda_device, event_ms, gpu_identity
from dmnerf_b200 import synth
from dmnerf_b200.testing import make_models
from dmnerf_b200.render import dm_nerf
from dmnerf_b200.embedder import get_embedder
from dmnerf_b200.helpers import get_select_full
from dmnerf_b200.evaluator import ins_criterion, img2mse
from dmnerf_b200.penalizer import ins_penalizer

dev = cuda_device("prof_full_iter.py")
ins_num = 13
wl = synth.workload("dmsr_study")
H, W = wl["H"], wl["W"]
nc, nf, _, _ = make_models(201, 202, ins_num, dev)
targs = types.SimpleNamespace(perturb=1.0, N_importance=128, is_train=True, N_ins=None, tolerance=0.05, deta_w=0.05)
pe, ve = get_embedder(10)[0], get_embedder(4)[0]
zc = torch.linspace(float(wl["near"]), float(wl["far"]), 64, device=dev)[None].expand(1024, 64)
nc.train(); nf.train()
_adam_kw = {"fused": True} if os.environ.get("ADAM", "") == "fused" else {}      # default: torch's choice (_foreach kernels), as train_dmsr.py
opt = torch.optim.Adam(list(nc.parameters()) + list(nf.parameters()), lr=5e-4, **_adam_kw)
gt_rgb = torch.rand(H, W, 3, device=dev)
gt_lab = (torch.arange(H * W, device=dev).reshape(H, W) * 7 // (H * W)).to(torch.int16)
pose = torch.from_numpy(wl["c2w"]).to(dev)
parts = os.environ.get("PARTS", "select,ins,pen").split(",")
tc0, ti0, rays0 = get_select_full(gt_rgb, pose, wl["K"], gt_lab, 1024)


def full_iteration():
    if "select" in parts:
        target_c, target_i, batch_rays = get_select_full(gt_rgb, pose, wl["K"], gt_lab, 1024)
    else:
        target_c, target_i, batch_rays = tc0, ti0, rays0
    info = dm_nerf(batch_rays, pe, ve, nc, nf, zc, targs)
    total = img2mse(info["rgb_coarse"], target_c) + img2mse(info["rgb_fine"], target_c)
    if "ins" in parts:
        total = total + ins_criterion(info["ins_coarse"], target_i, ins_num)[0] + ins_criterion(info["ins_fine"], target_i, ins_num)[0]
    if "pen" in parts:
        total = total + ins_penalizer(info["raw_coarse"], info["z_vals_coarse"], info["depth_coarse"], batch_rays[1], targs) \
            + ins_penalizer(info["raw_fine"], info["z_vals_fine"], info["depth_fine"], batch_rays[1], targs)
    opt.zero_grad()
    total.sum().backward()
    opt.step()


for _ in range(4):
    full_iteration()
torch.cuda.synchronize()
ms, _ = event_ms(lambda: [full_iteration() for _ in range(10)])
print("GPU: %s" % gpu_identity(dev)[1])
print("adam=%s " % os.environ.get("ADAM", "foreach (torch default)"), end="")
print("parts=%s: %.3f ms per iteration (CUDA events, 10 iterations back to back)" % (",".join(parts), ms / 10))
host = []
for _ in range(6):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    full_iteration()
    host.append(1e3 * (time.perf_counter() - t0))
    torch.cuda.synchronize()
print("host time to ISSUE one iteration (GPU idle at its start): %.3f ms (min of 6)" % min(host))
from torch.profiler import profile, ProfilerActivity      # noqa: E402
with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    for _ in range(3):
        full_iteration()
    torch.cuda.synchronize()
kern = {}
n_k = 0
for ev in prof.events():
    if str(ev.device_type).endswith("CUDA"):
        k = kern.setdefault(ev.name, [0.0, 0])
        k[0] += ev.device_time / 3.0; k[1] += 1; n_k += 1
rows = sorted(kern.items(), key=lambda r: -r[1][0])
tot = sum(v[0] for v in kern.values())
print("GPU-busy time per iteration: %.3f ms in %d kernels / copies" % (tot / 1e3, n_k // 3))
for k, (t, c) in rows[:int(os.environ.get("TOPN", "24"))]:
    print("%8.1f us  %5.1f%%  x%-3d %s" % (t, 100 * t / tot, c // 3, k[:120]))
