"""SURVEY section 8 row f4: the 256^3 density sweep of tools/mesh_generator.py:36-49 through the point-query entry point
(dmnerf_mlp_forward_points: points and zero view directions embedded inside the tensor-core kernel), timed on the device, plus
the CPU oracle on a bounded sample of the same points.      python tools/point_sweep.py [grid]"""
import sys
import time

import torch

from _harness import cuda_device, event_ms, gpu_identity
from dmnerf_b200 import synth
from dmnerf_b200.autograd import mlp_forward_points
from dmnerf_b200.engine import get_context
from dmnerf_b200.testing import make_models, raw_errs
from oracle import dmnerf_oracle as O

grid = int(sys.argv[1]) if len(sys.argv) > 1 else 256
dev = cuda_device("point_sweep.py")
_, nf, _, wf = make_models(101, 202, 13, dev)
t = torch.linspace(-3.0, 3.0, grid, device=dev)
chunk = grid * grid * 16                                      # 16 z-slabs per call (mesh_generator.py sweeps in chunks too)
sigma = torch.empty(grid ** 3, device=dev)
with torch.no_grad():
    def sweep():
        for z0 in range(0, grid, 16):
            zz = t[z0:z0 + 16]
            pts = torch.stack(torch.meshgrid(t, t, zz, indexing="ij"), -1).reshape(-1, 3)
            out = mlp_forward_points(nf, pts)
            sigma.view(grid, grid, grid)[:, :, z0:z0 + 16] = out[:, 3].view(grid, grid, -1)
    sweep()
    torch.cuda.synchronize()
    ms, _ = event_ms(sweep)
    get_context(dev).sync_check()
    n = grid ** 3
    flops = 2.0 * synth.macs_per_sample(13) * n
    print("GPU: %s" % gpu_identity(dev)[1])
    print("point query sweep: %d^3 = %d points in %.1f ms = %.1f M points/s, %.0f algorithmic TFLOP/s (incl. grid generation and the sigma scatter in torch)"
          % (grid, n, ms, n / ms / 1e3, flops / (ms * 1e-3) / 1e12))
    # CPU oracle on a sample of the same points
    sel = torch.randint(0, grid, (4096, 3), generator=torch.Generator().manual_seed(0))
    pts = torch.stack([t.cpu()[sel[:, 0]], t.cpu()[sel[:, 1]], t.cpu()[sel[:, 2]]], -1)
    x = torch.cat([O.embed(pts, 10), O.embed(torch.zeros_like(pts), 4)], -1)
    t0 = time.perf_counter()
    ref = O.mlp_forward(O.to_torch(wf), x)
    dt = time.perf_counter() - t0
    got = mlp_forward_points(nf, pts.to(dev)).cpu()
    print("CPU oracle: %.0f points/s (%d threads); parity on %d sampled points: scale-relative error %.2e"
          % (len(pts) / dt, torch.get_num_threads(), len(pts), max(raw_errs(got.numpy(), ref.numpy()))))
