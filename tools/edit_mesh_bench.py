#!/usr/bin/env python
"""Timing of meshing an edited scene (DESIGN.md, "Meshing an edited scene") at grid_dim 256: one JSON line with, per case
(ins_num 13 and 93, 1 and 3 moves, explicit boxes of 1/64 and 1/8 of the grid's points), the device time of the unedited
labelled sweep, of the edit pass (dmnerf_mesh_occupancy_edit) and of a whole edited_mesh, the target points evaluated, and the
GPU's name and power limit read in the same run.      python tools/edit_mesh_bench.py [--grid-dim 256] [--reps 2]

Synthetic trained-like networks (the bench.py ones), which need not cross the original's level 0.45 inside the grid: then the
level is the 90th percentile of the unedited occupancy (about 10 % of the grid solid).  The moved labels are those with the
most solid points, each translated by 2 voxels along a grid axis; the boxes are cubes of side dim / 4 and dim / 2 about the
grid's centre.  CUDA events, mean of --reps runs after one warm-up; the edit pass reads back its boxed point count once per slab and move, so its time includes those
round trips.  Nothing is written to disk."""
import argparse
import json

import numpy as np
import torch

from _harness import cuda_device, event_ms, gpu_identity
from dmnerf_b200 import objects as OB
from dmnerf_b200.testing import make_models

NEAR, FAR, N_IMPORTANCE, EXT = 4.0, 15.0, 128, (1.9, 7.0, 7.0)


def _timed(fn, reps):
    """(mean ms, result) of reps calls after one warm-up: the mean, not the median, is what DESIGN.md quotes of this bench."""
    fn()
    ms = []
    for _ in range(reps):
        t, out = event_ms(fn)
        ms.append(t)
    return float(np.mean(ms)), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid-dim", type=int, default=256)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    dev = cuda_device("edit_mesh_bench.py")
    dim = a.grid_dim
    T = np.eye(4)
    T[:3, 3] = (0.1, -0.2, 0.3)
    A, _ = OB.grid_affine(T, dim, EXT)
    cases = []
    for ins_num in (13, 93):
        _, nf, _, _ = make_models(101, 202, ins_num, dev)
        keep_all = OB.object_mask(ins_num, remove=[])
        with torch.no_grad():
            sweep_ms, (occ0, lab0) = _timed(lambda: OB.occupancy_objects(nf, T, keep_all, dim, EXT, NEAR, FAR, N_IMPORTANCE,
                                                                         device=dev), a.reps)
            sample = occ0.flatten()[::17]
            lo, hi = float(occ0.min()), float(occ0.max())
            level = 0.45 if lo < 0.45 < hi else float(sample.kthvalue(int(0.9 * sample.numel())).values)
            del sample
            solid = lab0[occ0 > level]
            k, c = torch.unique(solid, return_counts=True)
            top = [int(x) for x in k[torch.argsort(-c)][:3].tolist()]
            for n_moves in (1, 3):
                moves = []
                for i in range(n_moves):
                    shift = np.zeros(3)
                    shift[i % 3] = 2.0
                    m = np.eye(4)
                    m[:3, 3] = A @ shift                                       # 2 voxels along grid axis i
                    moves.append((top[i % len(top)], m))
                for frac, side in (("1/64", dim // 4), ("1/8", dim // 2)):
                    b0 = (dim - side) // 2
                    boxes = [(b0, b0 + side - 1) * 3] * n_moves

                    def edit():
                        occ, lab = occ0.clone(), lab0.clone()
                        return OB.edit_occupancy(nf, T, occ, lab, moves, boxes, EXT, level, NEAR, FAR, N_IMPORTANCE)
                    edit_ms, evaluated = _timed(edit, a.reps)
                    mesh_ms, m = _timed(lambda: OB.edited_mesh(nf, T, moves, dim, EXT, level, NEAR, FAR, N_IMPORTANCE, boxes=boxes),
                                        a.reps)
                    cases.append({"ins_num": ins_num, "level": level, "moves": n_moves, "box_fraction": frac,
                                  "labels": [mv for mv, _ in moves],
                                  "sweep_ms": sweep_ms, "edit_ms": edit_ms, "evaluated_points": evaluated,
                                  "evaluated_fraction": evaluated / dim ** 3, "edit_over_sweep": edit_ms / sweep_ms,
                                  "edited_mesh_ms": mesh_ms, "clean_vertices": int(m["clean_vertices"].shape[0])})
            del occ0, lab0
    name, smi, _ = gpu_identity(dev)
    print(json.dumps({"metric": "edited mesh device time", "grid_dim": dim, "reps": a.reps, "cases": cases,
                      "gpu": smi, "gpu_name": name,
                      "what": "unedited keep-all sweep, edit pass on a copy of it, whole edited_mesh (sweep + edit + marching "
                              "cubes + cleanup + vertex labels) with explicit boxes; synthetic trained-like networks; CUDA events, "
                              "mean of %d runs after one warm-up" % a.reps}))


if __name__ == "__main__":
    main()
