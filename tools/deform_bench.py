#!/usr/bin/env python
"""A deformed move against the rigid move of the same label and box (DESIGN.md, "Deforming objects"): one JSON line with, per
synthetic workload ("dmsr_study", ins_num 13, and "replica_room0_93", ins_num 93), the time of
  edit_pass     the edited sweep's edit pass (edit_occupancy on a copy of the keep-all sweep), grid_dim 256;
  edited_grid   the grid-only edit, grid_dim 256;
  render        render_frame(moves=) at 640x480;
and the GPU's name and power limit read in the same run.  The deformation twists the label's solid box by 60 degrees, tapers it
to 0.7 and bends it by a tenth of its height, 33 knots; the rigid move is the same translation without it.  Both variants share
the box, so both evaluate about the same targets; the difference is the fp64 pull of every grid point or sample.  Each pair
alternates within every round, timed on the host clock around a synchronised call; median of --reps rounds after --warmup.
    python tools/deform_bench.py [--reps 3] [--warmup 1]"""
import argparse
import json

import numpy as np
import torch

from _harness import alternate, cuda_device, gpu_identity, host_ms
from dmnerf_b200 import objects as OB
from dmnerf_b200 import synth
from dmnerf_b200.render import render_frame
from dmnerf_b200.testing import make_models

EXT, DIM, S, NI, CHUNK = (8.0, 8.0, 8.0), 256, 64, 128, 8192


def _pair(ms):
    med = {k: float(np.median(v)) for k, v in ms.items()}
    return {"ms": {k: [round(x, 2) for x in v] for k, v in ms.items()}, "ms_median": {k: round(v, 2) for k, v in med.items()},
            "deformed_over_rigid": round(med["deformed"] / med["rigid"], 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    dev = cuda_device("deform_bench.py")
    T = np.eye(4)
    A, b = OB.grid_affine(T, DIM, EXT)
    cases = []
    for wname in ("dmsr_study", "replica_room0_93"):
        w = synth.workload(wname)
        H, W, K, ins_num = w["H"], w["W"], np.asarray(w["K"], dtype=np.float32), w["ins_num"]
        near, far = float(w["near"]), float(w["far"])
        pose = torch.as_tensor(np.asarray(w["c2w"], dtype=np.float32), device=dev)
        nc, nf, _, _ = make_models(101, 202, ins_num, dev)
        with torch.no_grad():
            occ, labels = OB.occupancy_objects(nf, T, OB.object_mask(ins_num, remove=[]), DIM, EXT, near, far, NI, device=dev)
        sample = occ.flatten()[::17]
        sample = sample[sample > 0]
        level = 0.45 if float(occ.min()) < 0.45 < float(occ.max()) else float(sample.kthvalue(int(0.9 * sample.numel())).values)
        k, c = torch.unique(labels[occ > level], return_counts=True)
        label = int(k[torch.argmax(c)])
        m = np.eye(4)
        m[:3, 3] = A @ np.asarray([4.0, 0.0, 0.0])
        moves = [(label, m)]
        boxes = OB.edit_boxes(occ, labels, moves, T, EXT, level)
        box = boxes[0]
        lo, hi = A @ box[0::2].astype(np.float64) + b, A @ box[1::2].astype(np.float64) + b
        centre, up = (lo + hi) / 2, np.array([0.0, 0.0, 1.0])
        h = abs(hi[2] - lo[2]) / 2 or 1.0
        defs = [OB.deformation(centre, up, -h, h, 33, twist=lambda s: 60.0 * s, taper=lambda s: 1.0 - 0.3 * s,
                               bend=lambda s: 0.2 * h * s * s, bend_dir=(1.0, 0.0, 0.0))]
        case = {"workload": wname, "ins_num": ins_num, "label": label, "box": [int(v) for v in box], "level": level,
                "solid_voxels": int(c[k == label].sum())}
        with torch.no_grad():
            def edit(d):
                o, l_ = occ.clone(), labels.clone()
                return OB.edit_occupancy(nf, T, o, l_, moves, boxes, EXT, level, near, far, NI, deformations=d)
            case["evaluated"] = {"rigid": edit(None), "deformed": edit(defs)}
            case["edit_pass"] = _pair(alternate({"deformed": lambda: edit(defs), "rigid": lambda: edit(None)}, a.reps, a.warmup,
                                                clock=host_ms))
            case["edited_grid"] = _pair(alternate(
                {"deformed": lambda: OB.edited_grid(occ, labels, T, moves, EXT, level, boxes=boxes, deformations=defs),
                 "rigid": lambda: OB.edited_grid(occ, labels, T, moves, EXT, level, boxes=boxes)}, a.reps, a.warmup, clock=host_ms))
            md = OB.render_moves(occ, labels, T, moves, EXT, level, near, far, NI, boxes=boxes, deformations=defs)
            mr = OB.render_moves(occ, labels, T, moves, EXT, level, near, far, NI, boxes=boxes)
            case["render"] = _pair(alternate(
                {"deformed": lambda: render_frame(H, W, K, pose, near, far, nc, nf, N_samples=S, N_importance=NI, moves=md,
                                                  chunk=CHUNK, device=dev),
                 "rigid": lambda: render_frame(H, W, K, pose, near, far, nc, nf, N_samples=S, N_importance=NI, moves=mr, chunk=CHUNK,
                                               device=dev)}, a.reps, a.warmup, clock=host_ms))
        cases.append(case)
        del occ, labels
    name, smi, card = gpu_identity(dev)
    name, power = card or (name, "unknown")
    print(json.dumps({"bench": "deformed_vs_rigid", "gpu": name, "power_limit": power, "grid_dim": DIM, "frame": "640x480",
                      "chunk": CHUNK, "knots": 33, "reps": a.reps, "cases": cases}))


if __name__ == "__main__":
    main()
