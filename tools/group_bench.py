#!/usr/bin/env python
"""Groups against the same moves in sequence (DESIGN.md, "Moving objects together"): one JSON line with, per synthetic workload
("dmsr_study", ins_num 13, and "replica_room0_93", ins_num 93), the time of
  edited_grid   one move of a group of 2 labels against the 2 moves one label at a time, grid_dim 256 (the whole Python call,
                default boxes included);
  edited_sweep  the same pair, grid_dim 256 (the keep-all sweep and the edit passes);
  render        render_frame(moves=) at 640x480, the same pair;
and the GPU's name and power limit read in the same run.  These sweeps hold one or two solid labels, so each case says which
labels its group holds and how many solid voxels each has.  A group evaluates its targets in one pass over the union box, where
the sequence makes one pass per label.  Each pair alternates within every round, timed on the host clock around a synchronised
call; median of --reps rounds after --warmup.      python tools/group_bench.py [--reps 3] [--warmup 1]"""
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
            "group_over_sequence": round(med["group"] / med["sequence"], 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    dev = cuda_device("group_bench.py")
    T = np.eye(4)
    A, _ = OB.grid_affine(T, DIM, EXT)
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
        order = torch.argsort(c, descending=True)
        ks = [int(k[i]) for i in order[:2]]
        if len(ks) < 2:                                # one solid label: the second member is the next label, with no solid point
            ks.append((ks[0] + 1) % (ins_num + 1))
        solid = {str(x): int(c[k == x].sum()) for x in ks}
        m = np.eye(4)
        m[:3, 3] = A @ np.asarray([4.0, 0.0, 0.0])
        group, sequence = [(ks[0], m)], [(ks[0], m), (ks[1], m)]
        groups = [ks]
        case = {"workload": wname, "ins_num": ins_num, "group": ks, "solid_voxels": solid, "level": level}
        with torch.no_grad():
            case["edited_grid"] = _pair(alternate(
                {"group": lambda: OB.edited_grid(occ, labels, T, group, EXT, level, groups=groups),
                 "sequence": lambda: OB.edited_grid(occ, labels, T, sequence, EXT, level)}, a.reps, a.warmup, clock=host_ms))
            case["edited_sweep"] = _pair(alternate(
                {"group": lambda: OB.edited_sweep(nf, T, group, DIM, EXT, level, near, far, NI, groups=groups),
                 "sequence": lambda: OB.edited_sweep(nf, T, sequence, DIM, EXT, level, near, far, NI)}, a.reps, a.warmup,
                clock=host_ms))
            g = OB.render_moves(occ, labels, T, group, EXT, level, near, far, NI, groups=groups)
            s = OB.render_moves(occ, labels, T, sequence, EXT, level, near, far, NI)
            case["render"] = _pair(alternate(
                {"group": lambda: render_frame(H, W, K, pose, near, far, nc, nf, N_samples=S, N_importance=NI, moves=g, chunk=CHUNK,
                                               device=dev),
                 "sequence": lambda: render_frame(H, W, K, pose, near, far, nc, nf, N_samples=S, N_importance=NI, moves=s,
                                                  chunk=CHUNK, device=dev)}, a.reps, a.warmup, clock=host_ms))
        cases.append(case)
        del occ, labels
    name, smi, card = gpu_identity(dev)
    name, power = card or (name, "unknown")
    print(json.dumps({"bench": "group_vs_sequence", "gpu": name, "power_limit": power, "grid_dim": DIM, "frame": "640x480",
                      "chunk": CHUNK, "reps": a.reps, "cases": cases}))


if __name__ == "__main__":
    main()
