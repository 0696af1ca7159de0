#!/usr/bin/env python
"""Which objects a trained DM-NeRF checkpoint found, and where they are in 3-D (DESIGN.md, "Object inventory").

    python tools/find_objects.py CHECKPOINT.tar (--transform T [--extents X Y Z] | --poses POSES.npy --hwk H W K) [--trim 0]
                                 [--grid-dim 256] [--level 0.45] [--near 4 --far 15] [--out DIR]
                                 [--components {largest,split} [--connectivity {6,26}] [--min-voxels N]]

CHECKPOINT holds `network_coarse_state_dict` and `network_fine_state_dict`.  The grid is either given (--transform: a 4x4 as
.npy or 16 numbers of text, with --extents, default the original's 1.9 7 7) or found from the cameras (--poses: [N, 4, 4] or
[N, 3, 4] camera-to-world, --hwk: height, width and K as a .npy path or 9 numbers): the scene box of the fine network's solid
points inside the cameras' view, which --out then receives as scene_transform.txt and extents.txt for tools/extract_mesh.py
--extents.  Prints one JSON line: the box used and one entry per object (label, voxels, volume, centre, aabb, obb), all in the
network frame, the frame of the camera poses and of manipulator_eval's transforms.  --components splits each label into
connected components (DESIGN.md, "Connected components"): `largest` reports each object's largest component and adds its
label's component count and discarded voxels; `split` reports every component of at least --min-voxels voxels, with its id."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np   # noqa: E402


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("checkpoint")
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--transform", help="4x4 scene transform (.npy or text)")
    src.add_argument("--poses", help="camera-to-world poses [N, 4, 4] (.npy): find the scene box from the cameras")
    ap.add_argument("--hwk", nargs="+", metavar="H W K", help="with --poses: height, width and K (.npy file or 9 numbers)")
    ap.add_argument("--extents", type=float, nargs=3, default=[1.9, 7.0, 7.0], metavar=("X", "Y", "Z"))
    ap.add_argument("--trim", type=float, default=0.0, help="share of each object's points cut from each end of each axis")
    ap.add_argument("--grid-dim", type=int, default=256)
    ap.add_argument("--box-grid-dim", type=int, default=128, help="with --poses: the coarse sweep that finds the box")
    ap.add_argument("--level", type=float, default=0.45)
    ap.add_argument("--near", type=float, default=4.0)
    ap.add_argument("--far", type=float, default=15.0)
    ap.add_argument("--N-importance", type=int, default=128)
    ap.add_argument("--out", default=None)
    ap.add_argument("--components", choices=("largest", "split"), default=None,
                    help="split each label into connected components: its largest one, or every one")
    ap.add_argument("--connectivity", type=int, choices=(6, 26), default=None, help="with --components: 6 or 26 (default)")
    ap.add_argument("--min-voxels", type=int, default=None, help="with --components split: the smallest component reported")
    ap.add_argument("--device", default="cuda")
    a = ap.parse_args(argv)
    if a.components is None and a.connectivity is not None:
        ap.error("--connectivity needs --components")
    if a.min_voxels is not None and a.components != "split":
        ap.error("--min-voxels needs --components split")
    if a.min_voxels is not None and a.min_voxels < 1:
        ap.error("--min-voxels must be >= 1")
    if a.poses is not None:
        if not a.hwk or len(a.hwk) not in (3, 11):
            ap.error("--poses needs --hwk H W K (K as a .npy path or 9 numbers)")
        a.H, a.W = int(a.hwk[0]), int(a.hwk[1])
        a.K = (np.load(a.hwk[2]) if len(a.hwk) == 3 else np.array([float(v) for v in a.hwk[2:]])).astype(np.float64).reshape(3, 3)
    return a


def _json(e):
    out = {"label": e["label"], "voxels": e["voxels"], "volume": e["volume"], "centre": e["centre"].tolist(),
           "aabb": [e["aabb"][0].tolist(), e["aabb"][1].tolist()],
           "obb": {"centre": e["obb"]["centre"].tolist(), "axes": e["obb"]["axes"].tolist(),
                   "half_sizes": e["obb"]["half_sizes"].tolist()}}
    for k in ("component", "components", "discarded_voxels"):          # with --components
        if k in e:
            out[k] = e[k]
    return out


def components_args(a):
    """The component arguments of object_inventory for the parsed flags: none without --components."""
    if a.components is None:
        return {}
    return {"components": a.components, "connectivity": 26 if a.connectivity is None else a.connectivity,
            "min_voxels": 1 if a.min_voxels is None else a.min_voxels}


def main(argv=None):
    a = parse(argv)
    import torch
    from dmnerf_b200 import mesh as M
    from dmnerf_b200.objects import object_inventory, scene_box
    from dmnerf_b200.testing import model_from_weights
    ck = torch.load(a.checkpoint, map_location="cpu")
    nf = model_from_weights({k: v.float().numpy() for k, v in ck["network_fine_state_dict"].items()}, a.device)
    if a.poses is not None:
        poses = np.load(a.poses)
        T, ext = scene_box(nf, poses, (a.H, a.W, a.K), a.near, a.far, grid_dim=a.box_grid_dim, level=a.level,
                           N_importance=a.N_importance)
    else:
        T = np.load(a.transform) if a.transform.endswith(".npy") else np.loadtxt(a.transform)
        T, ext = M.check_transform(np.asarray(T, dtype=np.float64).reshape(4, 4)), np.asarray(a.extents, dtype=np.float64)
    inv = object_inventory(nf, T, tuple(ext), grid_dim=a.grid_dim, level=a.level, trim=a.trim, near=a.near, far=a.far,
                           N_importance=a.N_importance, **components_args(a))
    files = []
    if a.out is not None and a.poses is not None:
        os.makedirs(a.out, exist_ok=True)
        np.savetxt(os.path.join(a.out, "scene_transform.txt"), T, fmt="%.17g")
        np.savetxt(os.path.join(a.out, "extents.txt"), np.asarray(ext).reshape(1, 3), fmt="%.17g")
        files = ["scene_transform.txt", "extents.txt"]
    print(json.dumps({"scene_transform": np.asarray(T).tolist(), "extents": np.asarray(ext).tolist(), "trim": a.trim,
                      "objects": [_json(e) for e in inv], "files": files}))


if __name__ == "__main__":
    main()
