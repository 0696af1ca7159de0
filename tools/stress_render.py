"""Stress the fused render kernel for rare protocol stalls: many launches at several sizes, status word after every chunk.
    python tools/stress_render.py [launches]"""
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dmnerf_b200 import synth                            # noqa: E402
from dmnerf_b200.engine import get_context               # noqa: E402
from dmnerf_b200.testing import make_models              # noqa: E402
from dmnerf_b200.render import render_rays               # noqa: E402

launches = int(sys.argv[1]) if len(sys.argv) > 1 else 300
dev = "cuda"
slow = []
for name, n in (("dmsr_study", 132 * 2 * 8), ("replica_room0_93", 4096), ("dmsr_study", 1001)):
    wl = synth.workload(name)
    nc, nf, _, _ = make_models(101, 202, wl["ins_num"], dev)
    ro, rd = torch.from_numpy(wl["rays_o"][:n]).to(dev), torch.from_numpy(wl["rays_d"][:n]).to(dev)
    z = (torch.linspace(0, 1, 64) * (wl["far"] - wl["near"]) + wl["near"]).to(dev)
    with torch.no_grad():
        for i in range(launches):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = render_rays(ro, rd, nc, nf, z, want_raw=False, want_samples=False)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            if dt > 0.5:
                slow.append((name, n, i, dt))
            if i % 25 == 24:
                get_context(dev).sync_check()
    print(name, n, "ok", float(out["acc_fine"].mean()))
print("launches per size", launches, "slow:", slow[:10])
