#!/usr/bin/env python
"""Timing of object placement (DESIGN.md, "Object placement") at grid_dim 256: one JSON line with, per ins_num (13 and 93) and
lift (0 and grid_dim / 8), the device time of the keep-all labelled sweep, of placement_map as a whole and of its three stages
(column table, runs, map; kernel times from torch.profiler in a separate call), of place_object, the run and offset counts, and
the GPU's name and power limit read in the same run.
    python tools/place_bench.py [--grid-dim 256] [--reps 3]

Synthetic trained-like networks (the bench.py ones), which need not cross the original's level 0.45 inside the grid: then the
level is the 99th percentile of the sweep's occupancy (about 1 % of the grid solid; at the 90th percentile of
tools/collide_bench.py the label with the most points spans the grid and leaves one offset).  The placed label is the one with
the most solid points; down is the network's -y, the grid's fastest index axis (k) for the
identity rotation used here, the case where the column pass reads each column contiguously.  place_object aims at the grid's
centre and tests at most 64 offsets for stability.  The turned cases (DESIGN.md, "Turned placements") time, at lift 0, for the
label with the most points and for its piece inside an index cube of side grid_dim / 4 around its centre (a small object with
many offsets), placement_map against turned_placement_maps of 8 and of 36 turns and place_object(turns=8), with the 8-turn
call's stage split (torch.profiler) and its number of column-pass launches.  The arrangement cases (DESIGN.md, "Arranging
objects") time, against the sweep, edited_grid with 1 and with 8 moves (whole-voxel shifts of the labels with the most points) and
arrange_objects of 4 small pieces (each label's piece inside an index cube of side grid_dim / 4, as above) with turns=4, aimed at
four points around the grid's centre.  The calls are timed alternately (_harness.alternate, CUDA events, one warm-up round); each
ends in its read-back.  Nothing is written to disk."""
import argparse
import json

import numpy as np
import torch

from _harness import alternate, cuda_device, event_ms, gpu_identity
from dmnerf_b200 import objects as OB
from dmnerf_b200.testing import make_models

NEAR, FAR, N_IMPORTANCE, EXT = 4.0, 15.0, 128, (1.9, 7.0, 7.0)
DOWN = (0.0, -1.0, 0.0)
STAGES = {"column_table": ("grid_check_kernel", "place_column_kernel"),
          "moved_object": ("place_moved_kernel",),
          "runs": ("place_run_count_kernel", "DeviceScan", "place_run_write_kernel"),
          "map": ("place_map_kernel",)}


def _stats(ms):
    return {"mean_ms": float(np.mean(ms)), "min_ms": float(np.min(ms)), "max_ms": float(np.max(ms))}


def _stage_ms(fn, launches=None):
    """Device time per stage of one call of fn, from the kernel records of torch.profiler; launches (a dict) receives the
    number of column-pass launches."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {k: 0.0 for k in STAGES}
    columns = 0
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        columns += "place_column_kernel" in e.name
        for k, names in STAGES.items():
            if any(n in e.name for n in names):
                out[k] += e.device_time / 1e3
    if launches is not None:
        launches["column_pass"] = columns
    return out


def _small_piece(occ, lab, T, dim, level, label):
    """A small object with many offsets: the piece of `label` inside the index cube of side dim / 4 centred on the label's
    centre (the Region of that cube, applying to the label)."""
    _, _, centre = OB._object_extent((lab == label) & (occ > level))
    lo = [min(max(int(c) - dim // 8, 0), dim - dim // 4) for c in centre]
    cube = torch.zeros((dim,) * 3, dtype=torch.bool, device=occ.device)
    cube[lo[0]:lo[0] + dim // 4, lo[1]:lo[1] + dim // 4, lo[2]:lo[2] + dim // 4] = True
    return OB.region_from_mask(cube, T, EXT, applies=[label], outside="drop")


def turned_cases(occ, lab, T, dim, level, label, near, reps, what, piece=None):
    """The turned path for one object: placement_map against batched maps of 8 and 36 turns and place_object(turns=8)."""
    angles8, angles36 = [45.0 * k for k in range(8)], [10.0 * k for k in range(36)]
    case = {"label": label, "object": what, "level": level}
    kw = dict(extents=EXT, level=level, piece=piece)
    m = OB.placement_map(occ, lab, T, label, DOWN, 0, **kw)
    variants = {
        "placement_map": lambda: OB.placement_map(occ, lab, T, label, DOWN, 0, **kw),
        "turns_8": lambda: OB.turned_placement_maps(occ, lab, T, label, DOWN, angles8, 0, **kw),
        "turns_36": lambda: OB.turned_placement_maps(occ, lab, T, label, DOWN, angles36, 0, **kw),
        "place_object_turns_8": lambda: OB.place_object(occ, lab, T, label, DOWN, near, turns=8, **kw),
    }
    ms = alternate(variants, reps)
    launches = {}
    stages = [_stage_ms(lambda: OB.turned_placement_maps(occ, lab, T, label, DOWN, angles8, 0, **kw), launches)
              for _ in range(reps)]
    maps, unfit, unplaced = OB.turned_placement_maps(occ, lab, T, label, DOWN, angles8, 0, **kw)
    r = OB.place_object(occ, lab, T, label, DOWN, near, turns=8, **kw)
    case.update({"points": m["points"], "runs": m["runs"], "offsets": int(m["drop"].numel()),
                 "turns_8": {"mapped": len(maps), "unfit": unfit, "unplaced": unplaced,
                             "offsets": [int(x["drop"].numel()) for _, x in maps], "column_pass_launches": launches["column_pass"]},
                 "place_object_turns_8": {"candidates": r["candidates"], "tested": r["tested"], "turn": r["turn"]},
                 **{k + "_ms": _stats(v) for k, v in ms.items()},
                 **{"turns_8_stage_" + k + "_ms": _stats([s[k] for s in stages]) for k in STAGES}})
    return case


def arrange_cases(nf, keep_all, occ, lab, T, dim, level, reps, dev):
    """edited_grid of 1 and 8 moves and arrange_objects of 4 small pieces with turns=4, alternated with the sweep."""
    A, b = OB.grid_affine(T, dim, EXT)
    k, c = torch.unique(lab[occ > level], return_counts=True)
    labels = [int(x) for x in k[torch.argsort(c, descending=True)][:8]]
    moves = [(x, OB._translate(A @ np.array([(i % 3) - 1.0, 2.0, (i % 2) * 3.0]))) for i, x in enumerate(labels)]
    pieces = [_small_piece(occ, lab, T, dim, level, x) for x in labels[:4]]
    aims = [A @ np.array([dim / 2.0 + di, dim / 2.0, dim / 2.0 + dk]) + b for di, dk in ((-32, -32), (-32, 32), (32, -32), (32, 32))]
    items = [{"label": x, "near": y, "piece": pc, "turns": 4} for x, y, pc in zip(labels[:4], aims, pieces)]
    variants = {
        "sweep": lambda: OB.occupancy_objects(nf, T, keep_all, dim, EXT, NEAR, FAR, N_IMPORTANCE, device=dev),
        "edited_grid_1": lambda: OB.edited_grid(occ, lab, T, moves[:1], EXT, level),
        "edited_grid_8": lambda: OB.edited_grid(occ, lab, T, moves, EXT, level),
        "arrange_objects_4": lambda: OB.arrange_objects(occ, lab, T, items, DOWN, EXT, level),
    }
    ms = alternate(variants, reps)
    r = OB.arrange_objects(occ, lab, T, items, DOWN, EXT, level)
    return {"labels": labels, "level": level, "moves": len(moves),
            "arrange": [{"label": it["label"], "placed": it["placement"] is not None, "tested": it.get("tested"),
                         "turn": it.get("turn")} for it in r["items"]],
            **{k + "_ms": _stats(v) for k, v in ms.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid-dim", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    dev = cuda_device("place_bench.py")
    dim = a.grid_dim
    T = np.eye(4)
    T[:3, 3] = (0.1, -0.2, 0.3)
    A, b = OB.grid_affine(T, dim, EXT)
    near = A @ np.full(3, (dim - 1) / 2.0) + b
    cases, turned, arranged = [], [], []
    for ins_num in (13, 93):
        _, nf, _, _ = make_models(101, 202, ins_num, dev, trained_like=True)
        keep_all = OB.object_mask(ins_num, remove=[])
        with torch.no_grad():
            _, (occ, lab) = event_ms(lambda: OB.occupancy_objects(nf, T, keep_all, dim, EXT, NEAR, FAR, N_IMPORTANCE, device=dev))
            sample = occ.flatten()[::17]
            lo, hi = float(occ.min()), float(occ.max())
            level = 0.45 if lo < 0.45 < hi else float(sample.kthvalue(int(0.99 * sample.numel())).values)
            del sample
            k, c = torch.unique(lab[occ > level], return_counts=True)
            label = int(k[torch.argmax(c)])
            for lift in (0, dim // 8):
                case = {"ins_num": ins_num, "level": level, "label": label, "lift": lift}
                try:
                    m = OB.placement_map(occ, lab, T, label, DOWN, lift, EXT, level)
                except ValueError as e:                                  # the label's top leaves the grid at this lift
                    cases.append(dict(case, error=str(e)))
                    continue
                variants = {
                    "sweep": lambda: OB.occupancy_objects(nf, T, keep_all, dim, EXT, NEAR, FAR, N_IMPORTANCE, device=dev),
                    "placement_map": lambda: OB.placement_map(occ, lab, T, label, DOWN, lift, EXT, level),
                    "place_object": lambda: OB.place_object(occ, lab, T, label, DOWN, near, lift=lift, extents=EXT, level=level),
                }
                ms = alternate(variants, a.reps)
                stages = [_stage_ms(lambda: OB.placement_map(occ, lab, T, label, DOWN, lift, EXT, level)) for _ in range(a.reps)]
                r = OB.place_object(occ, lab, T, label, DOWN, near, lift=lift, extents=EXT, level=level)
                drop = m["drop"]
                case.update({"runs": m["runs"], "points": m["points"], "offsets": int(drop.numel()),
                             "blocked": int((drop < 0).sum()), "supported": int((m["support"] >= 0).sum()),
                             "place_object": {"candidates": r["candidates"], "tested": r["tested"],
                                              "found": r["placement"] is not None},
                             **{k + "_ms": _stats(v) for k, v in ms.items()},
                             **{"stage_" + k + "_ms": _stats([s[k] for s in stages]) for k in STAGES}})
                cases.append(case)
                del m, r
            turned.append(dict(turned_cases(occ, lab, T, dim, level, label, near, a.reps, "whole label"), ins_num=ins_num))
            piece = _small_piece(occ, lab, T, dim, level, label)
            turned.append(dict(turned_cases(occ, lab, T, dim, level, label, near, a.reps, "piece in a cube of side dim / 4", piece),
                               ins_num=ins_num))
            arranged.append(dict(arrange_cases(nf, keep_all, occ, lab, T, dim, level, a.reps, dev), ins_num=ins_num))
        del occ, lab
    name, smi, _ = gpu_identity(dev)
    print(json.dumps({"metric": "placement device time", "grid_dim": dim, "reps": a.reps, "down": DOWN, "cases": cases,
                      "turned": turned, "arrange": arranged, "gpu": smi,
                      "gpu_name": name,
                      "what": "keep-all labelled sweep, placement_map (stages: torch.profiler kernel times of one call each), "
                              "place_object (at most 64 stability tests); synthetic trained-like networks; CUDA events, "
                              "alternated, %d rounds after one warm-up" % a.reps}))


if __name__ == "__main__":
    main()
