#!/usr/bin/env python
"""Copies against moves (DESIGN.md, "Copying objects"): one JSON line with, per synthetic workload ("dmsr_study", ins_num 13, and
"replica_room0_93", ins_num 93), the time of
  edited_grid   one copy against the same move, grid_dim 256 (the whole Python call, default boxes included);
  edited_sweep  one copy against the same move, grid_dim 256 (the keep-all sweep and the edit pass);
  render        render_frame(moves=) at 640x480 with 1 and 4 copies against the same moves (the 4 are the one label translated
                along four directions, since these sweeps hold one or two solid labels);
and the GPU's name and power limit read in the same run.  A copy only skips the vacate, so the expectation is equal cost within
noise.  Each pair alternates within every round, timed on the host clock around a synchronised call; median of --reps rounds
after --warmup.      python tools/copy_bench.py [--reps 3] [--warmup 1]"""
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
            "copy_over_move": round(med["copy"] / med["move"], 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    dev = cuda_device("copy_bench.py")
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
        label = int(k[torch.argmax(c)])
        moves = []
        for shift in ([4.0, 0, 0], [0, 4.0, 0], [0, 0, 4.0], [-4.0, 0, 0]):
            m = np.eye(4)
            m[:3, 3] = A @ np.asarray(shift)
            moves.append((label, m))
        case = {"workload": wname, "ins_num": ins_num, "label": label, "level": level}
        with torch.no_grad():
            case["edited_grid"] = _pair(alternate(
                {"copy": lambda: OB.edited_grid(occ, labels, T, moves[:1], EXT, level, copies=True),
                 "move": lambda: OB.edited_grid(occ, labels, T, moves[:1], EXT, level)}, a.reps, a.warmup, clock=host_ms))
            case["edited_sweep"] = _pair(alternate(
                {"copy": lambda: OB.edited_sweep(nf, T, moves[:1], DIM, EXT, level, near, far, NI, copies=True),
                 "move": lambda: OB.edited_sweep(nf, T, moves[:1], DIM, EXT, level, near, far, NI)}, a.reps, a.warmup, clock=host_ms))
            for n in (1, 4):
                # a move of a label after a copy of it is rejected, and four moves of one label would each vacate the last one's
                # landing: the moves here are the same list with every flag off
                copied = OB.render_moves(occ, labels, T, moves[:n], EXT, level, near, far, NI, copies=True)
                moved = OB.render_moves(occ, labels, T, moves[:n], EXT, level, near, far, NI)
                case["render_%d" % n] = _pair(alternate(
                    {"copy": lambda m=copied: render_frame(H, W, K, pose, near, far, nc, nf, N_samples=S, N_importance=NI, moves=m,
                                                           chunk=CHUNK, device=dev),
                     "move": lambda m=moved: render_frame(H, W, K, pose, near, far, nc, nf, N_samples=S, N_importance=NI, moves=m,
                                                          chunk=CHUNK, device=dev)}, a.reps, a.warmup, clock=host_ms))
        cases.append(case)
        del occ, labels
    name, smi, card = gpu_identity(dev)
    name, power = card or (name, "unknown")
    print(json.dumps({"bench": "copy_vs_move", "gpu": name, "power_limit": power, "grid_dim": DIM, "frame": "640x480",
                      "chunk": CHUNK, "reps": a.reps, "cases": cases}))


if __name__ == "__main__":
    main()
