#!/usr/bin/env python
"""Timing of the collision checks (DESIGN.md, "Collision checks") at grid_dim 256: one JSON line with, per ins_num (13 and 93),
the device time of the keep-all labelled sweep, of move_overlap with one candidate, of a 1024-step slide_until_contact with a
box of 1/64 of the grid's points and of object_contacts, and the GPU's name and power limit read in the same run.
    python tools/collide_bench.py [--grid-dim 256] [--reps 3]

Synthetic trained-like networks (the bench.py ones), which need not cross the original's level 0.45 inside the grid: then the
level is the 90th percentile of the sweep's occupancy (about 10 % of the grid solid).  The moved label is the one with the most
solid points; the single candidate shifts it by 2 voxels along a grid axis; the slide moves it along that axis in steps of 1/8
voxel with the explicit box, a cube of side dim / 4 about the grid's centre, so that its work does not depend on the object's
size.  The checks are timed alternately (_harness.alternate, CUDA events, one warm-up round); each ends in its one read-back.
Nothing is written to disk."""
import argparse
import json

import numpy as np
import torch

from _harness import alternate, cuda_device, event_ms, gpu_identity
from dmnerf_b200 import objects as OB
from dmnerf_b200.testing import make_models

NEAR, FAR, N_IMPORTANCE, EXT = 4.0, 15.0, 128, (1.9, 7.0, 7.0)
SLIDE_STEPS = 1024


def _stats(ms):
    return {"mean_ms": float(np.mean(ms)), "min_ms": float(np.min(ms)), "max_ms": float(np.max(ms))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid-dim", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    dev = cuda_device("collide_bench.py")
    dim = a.grid_dim
    T = np.eye(4)
    T[:3, 3] = (0.1, -0.2, 0.3)
    A, _ = OB.grid_affine(T, dim, EXT)
    cases = []
    for ins_num in (13, 93):
        _, nf, _, _ = make_models(101, 202, ins_num, dev, trained_like=True)
        keep_all = OB.object_mask(ins_num, remove=[])
        with torch.no_grad():
            _, (occ, lab) = event_ms(lambda: OB.occupancy_objects(nf, T, keep_all, dim, EXT, NEAR, FAR, N_IMPORTANCE, device=dev))
            sample = occ.flatten()[::17]
            lo, hi = float(occ.min()), float(occ.max())
            level = 0.45 if lo < 0.45 < hi else float(sample.kthvalue(int(0.9 * sample.numel())).values)
            del sample
            k, c = torch.unique(lab[occ > level], return_counts=True)
            label = int(k[torch.argmax(c)])
            side = dim // 4
            b0 = (dim - side) // 2
            box = [(b0, b0 + side - 1) * 3]
            shift = np.eye(4)
            shift[:3, 3] = A @ np.array([2.0, 0.0, 0.0])
            step = float(np.linalg.norm(A[:, 0])) / 8                     # 1024 steps: 128 voxels
            variants = {
                "sweep": lambda: OB.occupancy_objects(nf, T, keep_all, dim, EXT, NEAR, FAR, N_IMPORTANCE, device=dev),
                "move_overlap_1": lambda: OB.move_overlap(occ, lab, T, [(label, shift)], EXT, level, boxes=box),
                # slide_until_contact's steps and answer, on the fixed box rather than the label's own solid box
                "slide_1024": lambda: OB.slide_result(*_slide(occ, lab, T, label, A[:, 0], step, level, box[0])),
                "object_contacts": lambda: OB.object_contacts(occ, lab, T, EXT, level),
            }
            ms = alternate(variants, a.reps)
            one = OB.move_overlap(occ, lab, T, [(label, shift)], EXT, level, boxes=box)[0]
            r = OB.slide_result(*_slide(occ, lab, T, label, A[:, 0], step, level, box[0]))
            cases.append({"ins_num": ins_num, "level": level, "label": label, "box_fraction": "1/64",
                          "move_overlap_1": {"landed": one["landed"], "total": one["total"]},
                          "slide": {"steps": len(r["steps"]), "distance": r["distance"]},
                          **{k + "_ms": _stats(v) for k, v in ms.items()}})
        del occ, lab
    name, smi, _ = gpu_identity(dev)
    print(json.dumps({"metric": "collision check device time", "grid_dim": dim, "reps": a.reps, "cases": cases, "gpu": smi,
                      "gpu_name": name,
                      "what": "keep-all labelled sweep, move_overlap with 1 candidate, slide_until_contact of %d steps (one "
                              "move_overlap call) with a 1/64 box, object_contacts; synthetic trained-like networks; CUDA events, "
                              "alternated, %d rounds after one warm-up" % (SLIDE_STEPS, a.reps)}))


def _slide(occ, lab, T, label, direction, step, level, box):
    d, s, mats = OB.slide_steps(direction, (SLIDE_STEPS - 1) * step, step)
    res = OB.move_overlap(occ, lab, T, [(label, m) for m in mats], EXT, level, boxes=[box] * len(mats))
    return d, s, res, 0


if __name__ == "__main__":
    main()
