#!/usr/bin/env python
"""Per-frame times of rendering moved objects (DESIGN.md, "Rendering moved objects") at 640x480: one JSON line with, per case
(synth.workload "dmsr_study", ins_num 13, and "replica_room0_93", ins_num 93; 1 and 3 moved labels), the time of
  (a) render_frame(moves=): the moves applied per sample inside the stage render, 8192 rays per chunk;
  (b) manipulate_frame with the same moves and N_test 4096: the exchanger, which renders the scene again per move;
  (c) the unedited stage render, render_rays(want_raw=True) over the same chunks: the floor of (a);
the targets (a) evaluated as a fraction of each pass's samples and the network passes per sample that follow, and the GPU's name and
power limit read in the same run.      python tools/render_moves_bench.py [--reps 2] [--warmup 1]

Synthetic trained-like networks (the bench.py ones).  The boxes come from a grid_dim 256 keep-all sweep of extents 8 about the
origin, where both cameras look.  The level is the first of 0.45 (when the sweep crosses it) and the 90th, 75th, 50th and 25th
percentiles of its positive occupancies at which the sweep holds 3 solid labels, so that the 3-move case moves 3 distinct
objects (the record lists the labels; a case with fewer distinct labels says so in distinct_labels).  The moved labels are
those with the most solid points, each translated by 4 voxels along a grid axis.  Variants alternate within each round, timed
on the host clock around a synchronised call.  (a) includes what (c) does not: the frame's rays and depths made on the device
and the maps copied to the host (render_frame returns host tensors), so its ratio over (c) slightly overstates the cost of the
edit.  Median of --reps rounds after --warmup."""
import argparse
import json
import types

import numpy as np
import torch

from _harness import alternate, cuda_device, gpu_identity, host_ms
from dmnerf_b200 import objects as OB
from dmnerf_b200 import synth
from dmnerf_b200.embedder import get_embedder
from dmnerf_b200.manipulator import manipulate_frame, rigid_rays
from dmnerf_b200.render import frame_rays, render_frame, render_rays
from dmnerf_b200.testing import make_models

EXT, DIM, S, NI, CHUNK = (8.0, 8.0, 8.0), 256, 64, 128, 8192


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    dev = cuda_device("render_moves_bench.py")
    T = np.eye(4)
    A, _ = OB.grid_affine(T, DIM, EXT)
    pe, ve = get_embedder(10)[0], get_embedder(4)[0]
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
            lo, hi = float(occ.min()), float(occ.max())
            levels = ([0.45] if lo < 0.45 < hi else []) + [float(sample.kthvalue(int(q * sample.numel())).values)
                                                           for q in (0.9, 0.75, 0.5, 0.25)]
            for level in levels:
                k, c = torch.unique(labels[occ > level], return_counts=True)
                top = [int(x) for x in k[torch.argsort(-c)][:3].tolist()]
                if len(top) == 3:
                    break
            ro, rd, z = frame_rays(H, W, K, pose, near, far, S, dev)
            for n_moves in (1, 3):
                moves = []
                for i in range(n_moves):
                    shift = np.zeros(3)
                    shift[i % 3] = 4.0
                    m = np.eye(4)
                    m[:3, 3] = A @ shift
                    moves.append((top[i % len(top)], m))
                moved = OB.render_moves(occ, labels, T, moves, EXT, level, near, far, NI)
                tars = [rigid_rays(H, W, K, m.astype(np.float32), pose) for _, m in moves]
                to, td = torch.stack([t[0] for t in tars]), torch.stack([t[1] for t in tars])
                args = types.SimpleNamespace(N_test=4096, near=near, far=far, N_samples=S, N_importance=NI, ins_num=ins_num,
                                             target_labels=[mv for mv, _ in moves])
                evaluated = []

                def moved_frame():
                    r = render_frame(H, W, K, pose, near, far, nc, nf, N_samples=S, N_importance=NI, moves=moved, chunk=CHUNK,
                                     device=dev)
                    evaluated[:] = r["evaluated"]

                def floor():
                    for b in range(0, H * W, CHUNK):
                        render_rays(ro[b:b + CHUNK], rd[b:b + CHUNK], nc, nf, z, N_importance=NI, want_raw=True)

                ms = alternate({"render_frame_moves": moved_frame,
                                "manipulate_frame": lambda: manipulate_frame(H, W, K, pose, to, td, pe, ve, nc, nf, args),
                                "stage_render": floor}, a.reps, a.warmup, clock=host_ms)
                med = {k: float(np.median(v)) for k, v in ms.items()}
                fc, ff = evaluated[0] / (H * W * S), evaluated[1] / (H * W * (S + NI))
                cases.append({"workload": wname, "ins_num": ins_num, "moves": n_moves, "labels": [mv for mv, _ in moves],
                              "distinct_labels": len(set(mv for mv, _ in moves)),
                              "level": level, "boxes": [list(b) for b in moved.boxes],
                              "ms": {k: [round(x, 1) for x in v] for k, v in ms.items()},
                              "ms_median": {k: round(v, 1) for k, v in med.items()},
                              "moves_over_stage": round(med["render_frame_moves"] / med["stage_render"], 3),
                              "exchanger_over_moves": round(med["manipulate_frame"] / med["render_frame_moves"], 2),
                              "evaluated": list(evaluated), "evaluated_fraction": {"coarse": round(fc, 4), "fine": round(ff, 4)},
                              "network_passes_per_sample": round(1.0 + (evaluated[0] + evaluated[1]) / (H * W * (2 * S + NI)), 4),
                              "exchanger_passes_per_sample": round((n_moves + 1) * (448 + 128 * n_moves) / (2 * S + NI), 2)})
            del occ, labels
    name, smi, card = gpu_identity(dev)
    name, power = card or (name, "unknown")
    print(json.dumps({"bench": "render_moves_640x480", "gpu": name, "power_limit": power, "grid_dim": DIM, "chunk": CHUNK,
                      "reps": a.reps, "cases": cases}))


if __name__ == "__main__":
    main()
