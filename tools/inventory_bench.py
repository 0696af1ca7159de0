#!/usr/bin/env python
"""Timing of the object inventory (dmnerf_b200.objects) at grid_dim 256: one JSON line with the device time of the selected
occupancy sweep with its label grid, of each inventory pass (voxels over the solid points, voxels inside the trimmed boxes,
spans), the whole inventory_from_grid call, and the GPU's name and power limit read in the same run, at ins_num 13 and 93.
        python tools/inventory_bench.py [--grid-dim 256] [--reps 3]

Every pass ends with its one device->host read (it synchronises), so a pass's time includes that read.  CUDA events around
each call, median of --reps after one warm-up.  Nothing is written to disk."""
import argparse
import json

import numpy as np
import torch

from _harness import cuda_device, event_ms, gpu_identity
from dmnerf_b200 import objects as OB
from dmnerf_b200.testing import make_models


def timed(fn, reps):
    """(result, median ms) of reps calls after one warm-up."""
    ms = []
    for _ in range(reps + 1):
        t, out = event_ms(fn)
        ms.append(t)
    return out, float(np.median(ms[1:]))


def one(ins_num, dim, reps, dev):
    nc, nf, _, _ = make_models(101, 202, ins_num, dev)            # the bench.py networks (synthetic, trained-like)
    T = np.eye(4)
    T[:3, 3] = (0.1, -0.2, 0.3)
    words = OB.object_mask(ins_num, remove=[ins_num])
    with torch.no_grad():
        (occ, labels), sweep = timed(lambda: OB.occupancy_objects(nf, T, words, dim, device=dev), reps)
        s = occ.flatten()[::17].float()
        level = 0.45 if float(occ.min()) < 0.45 < float(occ.max()) else float(s.kthvalue(int(0.98 * s.numel())).values)
        n = OB.MAX_LABELS
        (mom, hist), voxels = timed(lambda: OB.object_voxels(occ, labels, level, n), reps)
        boxes = OB.trimmed_boxes(hist, 0.01)
        _, voxels_boxed = timed(lambda: OB.object_voxels(occ, labels, level, n, boxes), reps)
        A, b = OB.grid_affine(T, dim)
        entries, axes = OB.describe_groups(mom, boxes, A, b, 1.0, range(ins_num))
        _, spans = timed(lambda: OB.object_spans(occ, labels, level, n, boxes, axes), reps)
        inv, total = timed(lambda: OB.inventory_from_grid(occ, labels, T, None, level, 0.01, range(ins_num)), reps)
    read = occ.numel() * (occ.element_size() + labels.element_size())
    return {"ins_num": ins_num, "level": level, "objects": len(inv), "solid_points": int(mom[:, 0].sum()),
            "ms": {"sweep": sweep, "voxels": voxels, "voxels_boxed": voxels_boxed, "spans": spans, "inventory_from_grid": total},
            "pass_read_GB_per_s": {k: read / (v * 1e-3) / 1e9 for k, v in (("voxels", voxels), ("spans", spans))}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid-dim", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    dev = cuda_device("inventory_bench.py")
    runs = [one(k, a.grid_dim, a.reps, dev) for k in (13, 93)]
    name, smi, _ = gpu_identity(dev)
    print(json.dumps({"metric": "object inventory device time", "grid_dim": a.grid_dim, "reps": a.reps, "runs": runs, "gpu": smi,
                      "gpu_name": name,
                      "what": "selected sweep with the label grid, then each pass over the occ (fp32) + label (int16) grids "
                              "with its read-back; trim 0.01; CUDA events, median of %d after one warm-up; GB/s = grid bytes "
                              "read once over the pass time" % a.reps}))


if __name__ == "__main__":
    main()
