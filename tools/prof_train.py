"""Kernel-level time breakdown of one training step (BASELINE config 4) with torch.profiler (CUPTI sees every kernel of the
process, including the native library's).  python tools/prof_train.py"""
import types

import numpy as np
import torch

from _harness import cuda_device, gpu_identity
from dmnerf_b200 import synth
from dmnerf_b200.testing import make_models
from dmnerf_b200.render import dm_nerf
from dmnerf_b200.embedder import get_embedder

dev = cuda_device("prof_train.py")
wl = synth.workload("dmsr_study")
nc, nf, _, _ = make_models(201, 202, 13, dev)
sel = np.random.Generator(np.random.PCG64(0)).choice(307200, 1024, replace=False)
ro, rd = torch.from_numpy(wl["rays_o"][sel]).to(dev), torch.from_numpy(wl["rays_d"][sel]).to(dev)
rays = torch.stack([ro, rd], 0)
targs = types.SimpleNamespace(perturb=1.0, N_importance=128, is_train=True, N_ins=None)
pe, ve = get_embedder(10)[0], get_embedder(4)[0]
zc = torch.linspace(float(wl["near"]), float(wl["far"]), 64, device=dev)[None].expand(1024, 64)
tgt = torch.rand(1024, 3, device=dev)
nc.train(); nf.train()
opt = torch.optim.Adam(list(nc.parameters()) + list(nf.parameters()), lr=5e-4)


def train_step():
    out = dm_nerf(rays, pe, ve, nc, nf, zc, targs)
    loss = ((out["rgb_fine"] - tgt) ** 2).mean() + ((out["rgb_coarse"] - tgt) ** 2).mean() + out["ins_fine"].mean()
    opt.zero_grad()
    loss.backward()
    opt.step()


for _ in range(3):
    train_step()
torch.cuda.synchronize()
from torch.profiler import profile, ProfilerActivity      # noqa: E402
with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    for _ in range(3):
        train_step()
    torch.cuda.synchronize()
rows = [(e.key, e.device_time_total / 3.0, e.count // 3) for e in prof.key_averages() if e.device_time_total > 0]
rows.sort(key=lambda r: -r[1])
tot = sum(r[1] for r in rows)
print("GPU: %s" % gpu_identity(dev)[1])
print("device time per step: %.2f ms over %d kernel kinds" % (tot / 1e3, len(rows)))
for k, t, c in rows[:28]:
    print("%8.1f us  %5.1f%%  x%-3d %s" % (t, 100 * t / tot, c, k[:110]))
