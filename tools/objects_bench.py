#!/usr/bin/env python
"""Cost of object selection on the device.  Prints one JSON line:
  * fused render kernel, one 640x480 frame (307 200 rays, 64 + 128 samples, deterministic), device-timed rays/s at ins_num 13
    (dmsr_study) and 93 (replica_room0_93): no selection, a keep-all mask, keep = {one label}, remove = {one label}.  The
    variants alternate inside every repetition, so they see the same clocks.
  * the selected occupancy sweep (with the label grid) and the per-object meshing stage at grid_dim 256, ins_num 13.
  * the GPU's name and power limit.
Synthetic trained-like networks (the bench.py ones).       python tools/objects_bench.py [--reps 3]"""
import argparse
import json

import numpy as np
import torch

from _harness import alternate, cuda_device, event_ms, gpu_identity
from dmnerf_b200 import synth
from dmnerf_b200 import mesh as M
from dmnerf_b200.helpers import z_val_sample
from dmnerf_b200.objects import meshes_from_labelled_grid, object_mask, occupancy_objects
from dmnerf_b200.render import render_rays
from dmnerf_b200.testing import make_models


def frame_rates(name, reps, dev):
    wl = synth.workload(name)
    ins_num = wl["ins_num"]
    nc, nf, _, _ = make_models(101, 202, ins_num, dev)
    ro, rd = torch.from_numpy(wl["rays_o"]).to(dev), torch.from_numpy(wl["rays_d"]).to(dev)
    z = z_val_sample(1, wl["near"], wl["far"], 64, device=dev)[0]
    n = ro.shape[0]
    with torch.no_grad():
        base = render_rays(ro, rd, nc, nf, z, want_raw=False, want_samples=False, want_coarse=False)
        lab = M.argmax_rows(base["ins_fine"])
        one = int(torch.bincount(lab, minlength=ins_num).argmax())          # the label most pixels show
        variants = {"none": None, "keep_all": list(range(ins_num + 1)), "keep_one": [one],
                    "remove_one": [k for k in range(ins_num + 1) if k != one]}
        run = {k: (lambda keep=keep: render_rays(ro, rd, nc, nf, z, want_raw=False, want_samples=False, want_coarse=False,
                                                 keep_objects=keep)) for k, keep in variants.items()}
        ms = alternate(run, reps)
    return {"ins_num": ins_num, "rays": n, "label": one,
            "rays_per_s": {k: n / (np.median(v) * 1e-3) for k, v in ms.items()},
            "ms": {k: [round(x, 3) for x in v] for k, v in ms.items()}}


def mesh_times(reps, dev, dim=256, ins_num=13):
    nc, nf, _, _ = make_models(101, 202, ins_num, dev)
    T = np.eye(4)
    T[:3, 3] = (0.1, -0.2, 0.3)
    near, far = 4.0, 15.0
    keep = object_mask(ins_num, remove=[ins_num])
    with torch.no_grad():
        occ, labels = occupancy_objects(nf, T, keep, dim, near=near, far=far, device=dev)
        sample = occ.flatten()[::17].float()
        lo, hi = float(occ.min()), float(occ.max())
        # as tools/mesh_bench.py: the original's level when the field crosses it, else the 99th percentile
        level = 0.45 if lo < 0.45 < hi else float(sample.kthvalue(int(0.99 * sample.numel())).values)
        objects = [k for k in torch.unique(labels).cpu().tolist() if k != ins_num]
        del occ, labels, sample
        sweep, per_obj, tris = [], [], None
        for _ in range(reps + 1):
            t_sweep, (occ, labels) = event_ms(lambda: occupancy_objects(nf, T, keep, dim, near=near, far=far, device=dev))
            t_mesh, meshes = event_ms(lambda: meshes_from_labelled_grid(occ, labels, T, objects, level))
            sweep.append(t_sweep)
            per_obj.append(t_mesh)
            tris = {k: int(m["clean_triangles"].shape[0]) for k, m in meshes.items()}
            del occ, labels, meshes                         # freed before the next timed sweep
    return {"grid_dim": dim, "ins_num": ins_num, "level": level, "objects": len(objects), "clean_triangles": tris,
            "sweep_ms": [round(x, 2) for x in sweep[1:]], "per_object_mesh_ms": [round(x, 2) for x in per_obj[1:]]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    dev = cuda_device("objects_bench.py")
    name, _, card = gpu_identity(dev)
    name, power = card or (name, "unknown")
    res = {"bench": "object_selection", "gpu": name, "power_limit": power,
           "frame_640x480": {wl: frame_rates(wl, a.reps, dev) for wl in ("dmsr_study", "replica_room0_93")},
           "mesh": mesh_times(a.reps, dev)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
