#!/usr/bin/env python
"""Timing of the connected components (dmnerf_b200.objects.object_components): one JSON line with the device time of
object_components at 6- and 26-connectivity, at each --grid-dims, on the labelled sweep of the bench networks at ins_num 13
and 93 and on a worst-case serpentine grid (one component whose union chains span the grid); the whole
inventory_from_grid(components="largest") against the sweep; and the GPU's name and power limit read in the same run.
        python tools/components_bench.py [--grid-dims 256 512] [--reps 3]

object_components ends with its read-backs (it synchronises), so its time includes them and the per-component table.  CUDA
events around each call, median of --reps after one warm-up; the sweep is timed once.  GB/s = the bytes of the occ (fp32) and
label (int16) grids over the call's time.  Nothing is written to disk."""
import argparse
import json

import numpy as np
import torch

from _harness import cuda_device, event_ms, gpu_identity
from dmnerf_b200 import objects as OB
from dmnerf_b200.testing import make_models
from oracle.components_oracle import serpentine


def timed(fn, reps):
    """(result, median ms) of reps calls after one warm-up; at reps 0 the time of the one cold call."""
    ms = []
    for _ in range(reps + 1):
        t, out = event_ms(fn)
        ms.append(t)
    return out, float(np.median(ms[1:] or ms))


def components(occ, labels, level, reps):
    read = occ.numel() * (occ.element_size() + (labels.element_size() if labels is not None else 0))
    out = {}
    for conn in (6, 26):
        cc, ms = timed(lambda: OB.object_components(occ, labels, level, conn), reps)
        out[str(conn)] = {"ms": ms, "components": int(cc["voxels"].shape[0]), "GB_per_s": read / (ms * 1e-3) / 1e9}
        del cc
    return out


def network(ins_num, dim, reps, dev):
    nc, nf, _, _ = make_models(101, 202, ins_num, dev)            # the bench.py networks (synthetic, trained-like)
    T = np.eye(4)
    T[:3, 3] = (0.1, -0.2, 0.3)
    words = OB.object_mask(ins_num, remove=[ins_num])
    with torch.no_grad():
        (occ, labels), sweep = timed(lambda: OB.occupancy_objects(nf, T, words, dim, device=dev), 0)
        s = occ.flatten()[::17].float()
        level = 0.45 if float(occ.min()) < 0.45 < float(occ.max()) else float(s.kthvalue(int(0.98 * s.numel())).values)
        res = {"ins_num": ins_num, "grid_dim": dim, "level": level, "solid_points": int((occ > level).sum()), "sweep_ms": sweep,
               "object_components": components(occ, labels, level, reps)}
        inv, ms = timed(lambda: OB.inventory_from_grid(occ, labels, T, None, level, 0.01, range(ins_num), components="largest"),
                        reps)
        _, plain = timed(lambda: OB.inventory_from_grid(occ, labels, T, None, level, 0.01, range(ins_num)), reps)
    res.update(objects=len(inv), inventory_largest_ms=ms, inventory_ms=plain, inventory_largest_share_of_sweep=ms / sweep)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid-dims", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    dev = cuda_device("components_bench.py")
    runs = []
    for dim in a.grid_dims:
        for k in (13, 93):
            runs.append(network(k, dim, a.reps, dev))
            torch.cuda.empty_cache()
        occ = torch.from_numpy(serpentine(dim)).to(dev)
        runs.append({"grid": "serpentine", "grid_dim": dim, "solid_points": int((occ > 0.45).sum()),
                     "object_components": components(occ, None, 0.45, a.reps)})
        del occ
        torch.cuda.empty_cache()
    name, smi, _ = gpu_identity(dev)
    print(json.dumps({"metric": "connected components device time", "reps": a.reps, "runs": runs, "gpu": smi, "gpu_name": name,
                      "what": "object_components (labelling, per-component table, read-backs) per connectivity; the whole "
                              "inventory_from_grid with components='largest' and without, trim 0.01, against one selected "
                              "sweep; CUDA events, median of %d after one warm-up; GB/s = occ + label grid bytes over the "
                              "call time" % a.reps}))


if __name__ == "__main__":
    main()
