"""Minimal driver for ncu: a few launches of the fused render kernel on one GPU."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dmnerf_b200 import synth                            # noqa: E402
from dmnerf_b200.engine import get_context               # noqa: E402
from dmnerf_b200.testing import make_models              # noqa: E402
from dmnerf_b200.render import render_rays               # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 132 * 2 * 96
dev = "cuda"
wl = synth.workload("dmsr_study")
nc, nf, _, _ = make_models(101, 202, wl["ins_num"], dev)
ro, rd = torch.from_numpy(wl["rays_o"][:n]).to(dev), torch.from_numpy(wl["rays_d"][:n]).to(dev)
z = (torch.linspace(0, 1, 64) * (wl["far"] - wl["near"]) + wl["near"]).to(dev)
with torch.no_grad():
    for _ in range(3):
        out = render_rays(ro, rd, nc, nf, z, want_raw=False, want_coarse=False, want_samples=False)
get_context(dev).sync_check()
print("done", n, float(out["acc_fine"].mean()))
