#!/usr/bin/env python
"""Render chosen objects of a trained DM-NeRF checkpoint: each one alone, or the scene without them.

    python tools/render_objects.py CHECKPOINT.tar --pose POSE.npy --hwk H W K (--keep L [L ...] | --remove L [L ...]) --out DIR
           [--near 4 --far 15 --N-samples 64 --N-importance 128]
           [(--no-floaters | --keep-piece ID [ID ...] | --drop-piece ID [ID ...]) --transform T [--extents X Y Z]
            [--grid-dim 256] [--level 0.45] [--connectivity {6,26}] [--dilate 1]]
           [--tint L R G B ...] [--opacity L S ...]

CHECKPOINT holds `network_coarse_state_dict` and `network_fine_state_dict` (the original's checkpoints).  POSE.npy holds one
camera-to-world pose [4, 4] (or [3, 4]) or several [N, 4, 4].  K is the 3x3 intrinsics, as a .npy file or as 9 numbers.  Writes
DIR/{i:03d}.png (RGBA: alpha = accumulated opacity, so an isolated object is a cut-out) and DIR/instance_{i:03d}.png (the
arg-max label; label k gets colour k of a fixed seeded palette).

Region selection (DESIGN.md, "Region selection") acts on the connected pieces of each object: one labelled occupancy sweep of the
fine network over the grid of --transform / --extents / --grid-dim (every label but the last, as tools/find_objects.py), split at
--level into --connectivity-connected components.  --no-floaters keeps each object's largest piece, --keep-piece keeps only the
given pieces of their objects, --drop-piece removes the given pieces and leaves the rest of their objects; a kept piece is grown
by --dilate voxels.  Piece IDs are the `component` ids of tools/find_objects.py --components split with the same sweep arguments.
A region combines with --keep / --remove, or stands alone (every label kept).

Object appearance (DESIGN.md, "Object appearance") changes how objects look: --tint L R G B gives label L the hue (R, G, B) and
keeps its shading (objects.tint; 1 1 1 is grey), --opacity L S scales label L's density by S >= 0 (0 removes it, below 1 fades
it, above 1 makes it more solid).  Both repeat, and combine with every flag above or stand alone."""
import argparse
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np   # noqa: E402


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("checkpoint")
    ap.add_argument("--pose", required=True)
    ap.add_argument("--hwk", nargs="+", required=True, metavar="H W K", help="height, width and K (.npy file or 9 numbers)")
    sel = ap.add_mutually_exclusive_group()
    sel.add_argument("--keep", type=int, nargs="+", metavar="L", help="render only these object labels")
    sel.add_argument("--remove", type=int, nargs="+", metavar="L", help="render the scene without these object labels")
    ap.add_argument("--out", required=True)
    ap.add_argument("--near", type=float, default=4.0)
    ap.add_argument("--far", type=float, default=15.0)
    ap.add_argument("--N-samples", type=int, default=64)
    ap.add_argument("--N-importance", type=int, default=128)
    ap.add_argument("--device", default="cuda")
    reg = ap.add_mutually_exclusive_group()
    reg.add_argument("--no-floaters", action="store_true", help="keep only each object's largest connected piece")
    reg.add_argument("--keep-piece", type=int, nargs="+", metavar="ID", help="keep only these pieces of their objects")
    reg.add_argument("--drop-piece", type=int, nargs="+", metavar="ID", help="remove these pieces, keep the rest of their objects")
    ap.add_argument("--transform", help="with a piece selection: 4x4 scene transform of the sweep grid (.npy or text)")
    ap.add_argument("--extents", type=float, nargs=3, default=[1.9, 7.0, 7.0], metavar=("X", "Y", "Z"))
    ap.add_argument("--grid-dim", type=int, default=256)
    ap.add_argument("--level", type=float, default=0.45)
    ap.add_argument("--connectivity", type=int, choices=(6, 26), default=26)
    ap.add_argument("--dilate", type=int, default=1, help="voxels a kept piece is grown by")
    ap.add_argument("--tint", type=float, nargs=4, action="append", default=[], metavar=("L", "R", "G", "B"),
                    help="give object label L the hue (R, G, B), keeping its shading (repeatable)")
    ap.add_argument("--opacity", type=float, nargs=2, action="append", default=[], metavar=("L", "S"),
                    help="scale object label L's density by S >= 0 (repeatable)")
    a = ap.parse_args(argv)
    a.region = "no_floaters" if a.no_floaters else ("keep" if a.keep_piece else ("drop" if a.drop_piece else None))
    if a.keep is None and a.remove is None and a.region is None and not a.tint and not a.opacity:
        ap.error("one of --keep, --remove, --no-floaters, --keep-piece, --drop-piece, --tint or --opacity is required")
    for flag, entries in (("--tint", a.tint), ("--opacity", a.opacity)):
        if any(e[0] != int(e[0]) for e in entries):
            ap.error("%s takes an integer label first" % flag)
    if any(not s >= 0 for _, s in a.opacity):
        ap.error("--opacity S must be >= 0")
    a.tint = {int(e[0]): tuple(e[1:]) for e in a.tint}
    a.opacity = {int(e[0]): e[1] for e in a.opacity}
    if a.region is not None and a.transform is None:
        ap.error("a piece selection needs --transform (the sweep grid)")
    if a.dilate < 0:
        ap.error("--dilate must be >= 0")
    if len(a.hwk) not in (3, 11):
        ap.error("--hwk takes H W and K as a .npy path or as 9 numbers")
    a.H, a.W = int(a.hwk[0]), int(a.hwk[1])
    a.K = (np.load(a.hwk[2]) if len(a.hwk) == 3 else np.array([float(v) for v in a.hwk[2:]])).astype(np.float32).reshape(3, 3)
    return a


def piece_region(a, model_fine):
    """The Region of the piece flags: the labelled sweep of every label but ins_num, its components, then component_region."""
    import torch
    from dmnerf_b200 import mesh as M
    from dmnerf_b200.objects import (component_region, largest_components, object_components, object_mask,
                                     occupancy_objects)
    T = np.load(a.transform) if a.transform.endswith(".npy") else np.loadtxt(a.transform)
    T, ext = M.check_transform(np.asarray(T, dtype=np.float64).reshape(4, 4)), tuple(a.extents)
    ins_num = int(model_fine.ins_linear.weight.shape[0]) - 1
    with torch.no_grad():
        occ, labels = occupancy_objects(model_fine, T, object_mask(ins_num, keep=range(ins_num)), a.grid_dim, ext, a.near, a.far,
                                        a.N_importance, device=next(model_fine.parameters()).device)
        cc = object_components(occ, labels, a.level, a.connectivity)
    del occ, labels
    if a.region == "no_floaters":
        best = largest_components(cc["label"], cc["voxels"])
        ids = [best[k] for k in sorted(best) if k != ins_num]
    else:
        ids = a.keep_piece if a.region == "keep" else a.drop_piece
    return component_region(cc, ids, T, ext, dilate=a.dilate, connectivity=a.connectivity, invert=a.region == "drop")


def main(argv=None):
    a = parse(argv)
    import torch
    from dmnerf_b200.embedder import get_embedder
    from dmnerf_b200.objects import Appearance, render_objects, tint
    from dmnerf_b200.testing import model_from_weights
    ck = torch.load(a.checkpoint, map_location="cpu")
    nets = [model_from_weights({k: v.float().numpy() for k, v in ck[key].items()}, a.device)
            for key in ("network_coarse_state_dict", "network_fine_state_dict")]
    poses = np.load(a.pose).astype(np.float32)
    if poses.ndim == 2:
        poses = poses[None]
    pe, _ = get_embedder(10)
    ve, _ = get_embedder(4)
    args = types.SimpleNamespace(near=a.near, far=a.far, N_samples=a.N_samples, N_importance=a.N_importance)
    region = piece_region(a, nets[1]) if a.region is not None else None
    appearance = None
    if a.tint or a.opacity:
        ins_num = int(nets[1].ins_linear.weight.shape[0]) - 1
        appearance = Appearance(ins_num, colour={k: tint(rgb) for k, rgb in a.tint.items()}, density=a.opacity)
    maps = render_objects(pe, ve, nets[0], nets[1], poses, (a.H, a.W, a.K), args, keep=a.keep, remove=a.remove, savedir=a.out,
                          region=region, appearance=appearance)
    print(json.dumps({"frames": len(maps), "mean_acc": [float(m["acc"].mean()) for m in maps],
                      "files": sorted(os.listdir(a.out))}))


if __name__ == "__main__":
    main()
