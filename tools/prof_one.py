"""Minimal driver for a profiler: a few launches of the fine-network tensor-core kernel (rays mode) on one GPU."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dmnerf_b200 import synth, _lib                      # noqa: E402
from dmnerf_b200.engine import get_context               # noqa: E402
from dmnerf_b200.testing import model_from_weights       # noqa: E402
from dmnerf_b200.autograd import mlp_forward_rays        # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 132 * 256
dev = "cuda"
wl = synth.workload("dmsr_study")
net = model_from_weights(synth.make_weights(202, 13), dev).eval()
ro, rd = torch.from_numpy(wl["rays_o"][:n]).to(dev), torch.from_numpy(wl["rays_d"][:n]).to(dev)
z = (torch.rand(n, 192, device=dev).sort(-1).values * 11 + 4).contiguous()
with torch.no_grad():
    for _ in range(3):
        mlp_forward_rays(net, ro, rd, z, _lib.IMPL_UMMA)
get_context(dev).sync_check()
print("done", n)
