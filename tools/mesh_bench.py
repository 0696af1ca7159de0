#!/usr/bin/env python
"""Timing of labelled mesh extraction (dmnerf_b200.mesh, the original's mesh_main) at grid_dim 256: one JSON line with the
device time of each stage (occupancy sweep / marching cubes / normals + cleanup / label rays), the vertex and triangle counts,
the sweep's points/s and algorithmic TFLOP/s (2 x synth.macs_per_sample per grid point), and the GPU's name and power limit read
in the same run.      python tools/mesh_bench.py [--grid-dim 256] [--ins-num 13] [--reps 2]

Each stage is timed with CUDA events around its calls, mean of --reps runs after one warm-up.  Marching cubes and the cleanup
read their counts back (one synchronisation each), so their times include that round trip.  Nothing is written to disk."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dmnerf_b200 import mesh as M, synth                      # noqa: E402
from dmnerf_b200.testing import make_models                   # noqa: E402

N_SAMPLES, N_IMPORTANCE, N_TEST, MIN_CLUSTER = 64, 128, 4096, 400      # mesh_main's defaults (configs/dmsr/test/meshing.txt)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid-dim", type=int, default=256)
    ap.add_argument("--ins-num", type=int, default=13)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "tools/mesh_bench.py needs a CUDA device; there is no CPU fallback"
    dev = torch.device("cuda", 0)
    nc, nf, _, _ = make_models(101, 202, a.ins_num, dev)          # the bench.py networks (synthetic, trained-like)
    T = np.eye(4)
    T[:3, 3] = (0.1, -0.2, 0.3)
    dim, near, far = a.grid_dim, 4.0, 15.0
    with torch.no_grad():
        # the synthetic networks need not cross the original's level 0.45 inside the grid: then the level is the 99th percentile
        # of the occupancy (about 1% of the grid inside), so that every stage has a surface to work on
        occ = M.occupancy_grid(nf, T, dim, near=near, far=far, N_importance=N_IMPORTANCE, device=dev)
        lo, hi = float(occ.min()), float(occ.max())
        sample = occ.flatten()[::17].float()
        level = 0.45 if lo < 0.45 < hi else float(sample.kthvalue(int(0.99 * sample.numel())).values)
        del occ, sample

        def run():
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
            ev[0].record()
            occ = M.occupancy_grid(nf, T, dim, near=near, far=far, N_importance=N_IMPORTANCE, device=dev)
            ev[1].record()
            v_idx, tris = M.marching_cubes(occ, level)
            ev[2].record()
            verts = M.to_scene(v_idx, T, dim)
            normals = M.vertex_normals(verts, tris)
            cv, cn, ct = M.clean_mesh(verts, normals, tris, MIN_CLUSTER)
            ev[3].record()
            ro, rd = M.label_rays(cv, cn, near)
            M.render_labels(nc, nf, ro, rd, N_SAMPLES, N_IMPORTANCE, N_TEST)
            ev[4].record()
            torch.cuda.synchronize(dev)
            return [ev[i].elapsed_time(ev[i + 1]) for i in range(4)], (verts.shape[0], tris.shape[0], cv.shape[0], ct.shape[0])

        run()
        times = []
        for _ in range(a.reps):
            ms, counts = run()
            times.append(ms)
    ms = np.mean(np.array(times), 0)
    n_pts = dim ** 3
    flops = 2.0 * synth.macs_per_sample(a.ins_num) * n_pts
    try:
        gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as exc:
        gpu = "nvidia-smi unavailable: %s" % exc
    print(json.dumps({
        "metric": "mesh extraction device time", "grid_dim": dim, "ins_num": a.ins_num, "reps": a.reps, "level": level,
        "occupancy_range": [lo, hi],
        "ms": {"sweep": ms[0], "marching_cubes": ms[1], "normals_cleanup": ms[2], "label_rays": ms[3], "total": float(ms.sum())},
        "vertices": counts[0], "triangles": counts[1], "clean_vertices": counts[2], "clean_triangles": counts[3],
        "sweep_points_per_s": n_pts / (ms[0] * 1e-3), "sweep_tflops": flops / (ms[0] * 1e-3) / 1e12,
        "label_rays_per_s": counts[2] / (ms[3] * 1e-3) if ms[3] > 0 else None,
        "gpu": gpu, "gpu_name": torch.cuda.get_device_name(dev),
        "what": "mesh_main defaults (level 0.45 unless the occupancy does not cross it, extents 1.9 x 7 x 7, near 4, far 15, "
                "64 + 128 samples, N_test 4096, clusters >= 400) on synthetic trained-like networks; CUDA events, mean of %d runs "
                "after one warm-up; sweep TFLOP/s = 2 x macs_per_sample x grid points over the sweep time (algorithmic)" % a.reps}))


if __name__ == "__main__":
    main()
