#!/usr/bin/env python
"""Timing of labelled mesh extraction (dmnerf_b200.mesh, the original's mesh_main) at grid_dim 256: one JSON line with the
device time of each stage (occupancy sweep / marching cubes / normals + cleanup / label rays), the vertex and triangle counts,
the sweep's points/s and algorithmic TFLOP/s (2 x synth.macs_per_sample per grid point), and the GPU's name and power limit read
in the same run.      python tools/mesh_bench.py [--grid-dim 256] [--ins-num 13] [--reps 2]

Each stage is timed with CUDA events around its calls, mean of --reps runs after one warm-up.  Marching cubes and the cleanup
read their counts back (one synchronisation each), so their times include that round trip.  Nothing is written to disk."""
import argparse
import json

import numpy as np
import torch

from _harness import cuda_device, gpu_identity, stages_ms
from dmnerf_b200 import mesh as M, synth
from dmnerf_b200.testing import make_models

N_SAMPLES, N_IMPORTANCE, N_TEST, MIN_CLUSTER = 64, 128, 4096, 400      # mesh_main's defaults (configs/dmsr/test/meshing.txt)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid-dim", type=int, default=256)
    ap.add_argument("--ins-num", type=int, default=13)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    dev = cuda_device("mesh_bench.py")
    nc, nf, _, _ = make_models(101, 202, a.ins_num, dev)          # the bench.py networks (synthetic, trained-like)
    T = np.eye(4)
    T[:3, 3] = (0.1, -0.2, 0.3)
    dim, near, far = a.grid_dim, 4.0, 15.0

    def sweep():
        return M.occupancy_grid(nf, T, dim, near=near, far=far, N_importance=N_IMPORTANCE, device=dev)

    def cleanup(mc):
        v_idx, tris = mc
        verts = M.to_scene(v_idx, T, dim)
        return verts, M.clean_mesh(verts, M.vertex_normals(verts, tris), tris, MIN_CLUSTER)

    def label_rays(mesh):
        _, (cv, cn, _) = mesh
        ro, rd = M.label_rays(cv, cn, near)
        M.render_labels(nc, nf, ro, rd, N_SAMPLES, N_IMPORTANCE, N_TEST)

    def run():
        # the four stages back to back with one event between each and one synchronise at the end
        ms, (_, (_, tris), (verts, (cv, _, ct)), _) = stages_ms(sweep, lambda occ: M.marching_cubes(occ, level), cleanup,
                                                                label_rays)
        return ms, (verts.shape[0], tris.shape[0], cv.shape[0], ct.shape[0])

    with torch.no_grad():
        # the synthetic networks need not cross the original's level 0.45 inside the grid: then the level is the 99th percentile
        # of the occupancy (about 1% of the grid inside), so that every stage has a surface to work on
        occ = sweep()
        lo, hi = float(occ.min()), float(occ.max())
        sample = occ.flatten()[::17].float()
        level = 0.45 if lo < 0.45 < hi else float(sample.kthvalue(int(0.99 * sample.numel())).values)
        del occ, sample
        run()
        times = []
        for _ in range(a.reps):
            ms, counts = run()
            times.append(ms)
    ms = np.mean(np.array(times), 0)
    n_pts = dim ** 3
    flops = 2.0 * synth.macs_per_sample(a.ins_num) * n_pts
    name, smi, _ = gpu_identity(dev)
    print(json.dumps({
        "metric": "mesh extraction device time", "grid_dim": dim, "ins_num": a.ins_num, "reps": a.reps, "level": level,
        "occupancy_range": [lo, hi],
        "ms": {"sweep": ms[0], "marching_cubes": ms[1], "normals_cleanup": ms[2], "label_rays": ms[3], "total": float(ms.sum())},
        "vertices": counts[0], "triangles": counts[1], "clean_vertices": counts[2], "clean_triangles": counts[3],
        "sweep_points_per_s": n_pts / (ms[0] * 1e-3), "sweep_tflops": flops / (ms[0] * 1e-3) / 1e12,
        "label_rays_per_s": counts[2] / (ms[3] * 1e-3) if ms[3] > 0 else None,
        "gpu": smi, "gpu_name": name,
        "what": "mesh_main defaults (level 0.45 unless the occupancy does not cross it, extents 1.9 x 7 x 7, near 4, far 15, "
                "64 + 128 samples, N_test 4096, clusters >= 400) on synthetic trained-like networks; CUDA events, mean of %d runs "
                "after one warm-up; sweep TFLOP/s = 2 x macs_per_sample x grid points over the sweep time (algorithmic)" % a.reps}))


if __name__ == "__main__":
    main()
