#!/usr/bin/env python
"""Labelled object mesh of a trained DM-NeRF checkpoint, without trimesh, skimage or open3d.

    python tools/extract_mesh.py CHECKPOINT.tar TRANSFORM --out DIR [--name NAME] [--grid-dim 256] [--extents 1.9 7 7] ...

CHECKPOINT holds `network_coarse_state_dict` and `network_fine_state_dict` (the original's checkpoints).  TRANSFORM is the 4x4
scene transform, inv(to_origin) of the scene mesh's oriented bounds, as a .npy file or as text (16 numbers).  Writes
DIR/NAME.ply (the marching-cubes mesh in scene space) and DIR/color_NAME.ply (cleaned, every vertex coloured by its object label).
Without --color-dict (JSON: label -> colour index) and --palette (.npy [K, 3] uint8), label k gets colour k of a fixed
seeded palette.  --per-object also writes DIR/NAME_obj{k}.ply for every object k: the cleaned mesh of that object alone, from
a selected occupancy sweep whose grid points are labelled by the network (closed wherever the object does not touch the grid
boundary); --objects limits it to the labels given, and --largest-component meshes each object's largest connected component
alone (DESIGN.md, "Connected components")."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np   # noqa: E402
import torch         # noqa: E402


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("checkpoint")
    ap.add_argument("transform")
    ap.add_argument("--out", required=True)
    ap.add_argument("--name", default="mesh")
    ap.add_argument("--grid-dim", type=int, default=256)
    ap.add_argument("--extents", type=float, nargs=3, default=[1.9, 7.0, 7.0], metavar=("X", "Y", "Z"),
                    help="grid size along the transform's axes (default: the original's 1.9 7 7; tools/find_objects.py "
                         "writes the found box's)")
    ap.add_argument("--near", type=float, default=4.0)
    ap.add_argument("--far", type=float, default=15.0)
    ap.add_argument("--N-samples", type=int, default=64)
    ap.add_argument("--N-importance", type=int, default=128)
    ap.add_argument("--N-test", type=int, default=4096)
    ap.add_argument("--min-cluster", type=int, default=400)
    ap.add_argument("--color-dict", default=None)
    ap.add_argument("--palette", default=None)
    ap.add_argument("--per-object", action="store_true", help="also write NAME_obj{k}.ply, one mesh per object")
    ap.add_argument("--objects", type=int, nargs="+", default=None, help="with --per-object: only these labels")
    ap.add_argument("--largest-component", action="store_true",
                    help="with --per-object: mesh each object's largest connected component only")
    ap.add_argument("--device", default="cuda")
    a = ap.parse_args(argv)
    if a.largest_component and not a.per_object:
        ap.error("--largest-component needs --per-object")
    return a


def main(argv=None):
    a = parse(argv)

    from dmnerf_b200 import mesh as M
    from dmnerf_b200.testing import model_from_weights
    T = np.load(a.transform) if a.transform.endswith(".npy") else np.loadtxt(a.transform)
    T = M.check_transform(np.asarray(T, dtype=np.float64).reshape(4, 4))
    ck = torch.load(a.checkpoint, map_location="cpu")
    nets = [model_from_weights({k: v.float().numpy() for k, v in ck[key].items()}, a.device)
            for key in ("network_coarse_state_dict", "network_fine_state_dict")]
    ins_num = nets[1].ins_linear.weight.shape[0] - 1
    out = M.extract_mesh(nets[1], nets[0], T, grid_dim=a.grid_dim, extents=tuple(a.extents), near=a.near, far=a.far, N_samples=a.N_samples,
                         N_importance=a.N_importance, N_test=a.N_test, min_cluster=a.min_cluster)
    os.makedirs(a.out, exist_ok=True)
    M.write_ply(os.path.join(a.out, a.name + ".ply"), out["vertices"], out["triangles"])
    labels = out["labels"].cpu().numpy()
    n_col = int(max(ins_num, labels.max(initial=0))) + 1
    palette = np.load(a.palette) if a.palette else np.random.default_rng(0).integers(0, 256, (n_col, 3))
    color_dict = json.load(open(a.color_dict)) if a.color_dict else {str(k): k for k in range(len(palette))}
    ins_map = {str(k): k for k in range(n_col)}
    colors = M.label_colors(labels, palette, color_dict, ins_map)
    M.write_ply(os.path.join(a.out, "color_" + a.name + ".ply"), out["clean_vertices"], out["clean_triangles"], colors)
    files = [a.name + ".ply", "color_" + a.name + ".ply"]
    per_object = {}
    if a.per_object:
        from dmnerf_b200.objects import object_meshes
        meshes = object_meshes(nets[1], nets[0], T, objects=a.objects, grid_dim=a.grid_dim, extents=tuple(a.extents), near=a.near, far=a.far,
                               N_importance=a.N_importance, min_cluster=a.min_cluster,
                               components="largest" if a.largest_component else None)
        for k, m in meshes.items():
            name = "%s_obj%d.ply" % (a.name, k)
            M.write_ply(os.path.join(a.out, name), m["clean_vertices"], m["clean_triangles"])
            files.append(name)
            per_object[str(k)] = int(m["clean_triangles"].shape[0])
    res = {"vertices": int(out["vertices"].shape[0]), "triangles": int(out["triangles"].shape[0]),
           "clean_vertices": int(out["clean_vertices"].shape[0]), "clean_triangles": int(out["clean_triangles"].shape[0]),
           "files": files}
    if a.per_object:
        res["object_triangles"] = per_object
    print(json.dumps(res))


if __name__ == "__main__":
    main()
