#!/usr/bin/env python
"""Labelled object mesh of a trained DM-NeRF checkpoint, without trimesh, skimage or open3d.

    python tools/extract_mesh.py CHECKPOINT.tar TRANSFORM --out DIR [--name NAME] [--grid-dim 256] [--near 4 --far 15] ...

CHECKPOINT holds `network_coarse_state_dict` and `network_fine_state_dict` (the original's checkpoints).  TRANSFORM is the 4x4
scene transform, inv(to_origin) of the scene mesh's oriented bounds, as a .npy file or as text (16 numbers).  Writes
DIR/NAME.ply (the marching-cubes mesh in scene space) and DIR/color_NAME.ply (cleaned, every vertex coloured by its object label).
Without --color-dict (JSON: label -> colour index) and --palette (.npy [K, 3] uint8), label k gets colour k of a fixed
seeded palette."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np   # noqa: E402
import torch         # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("checkpoint")
    ap.add_argument("transform")
    ap.add_argument("--out", required=True)
    ap.add_argument("--name", default="mesh")
    ap.add_argument("--grid-dim", type=int, default=256)
    ap.add_argument("--near", type=float, default=4.0)
    ap.add_argument("--far", type=float, default=15.0)
    ap.add_argument("--N-samples", type=int, default=64)
    ap.add_argument("--N-importance", type=int, default=128)
    ap.add_argument("--N-test", type=int, default=4096)
    ap.add_argument("--min-cluster", type=int, default=400)
    ap.add_argument("--color-dict", default=None)
    ap.add_argument("--palette", default=None)
    ap.add_argument("--device", default="cuda")
    a = ap.parse_args(argv)

    from dmnerf_b200 import mesh as M
    from dmnerf_b200.testing import model_from_weights
    T = np.load(a.transform) if a.transform.endswith(".npy") else np.loadtxt(a.transform)
    T = M.check_transform(np.asarray(T, dtype=np.float64).reshape(4, 4))
    ck = torch.load(a.checkpoint, map_location="cpu")
    nets = [model_from_weights({k: v.float().numpy() for k, v in ck[key].items()}, a.device)
            for key in ("network_coarse_state_dict", "network_fine_state_dict")]
    ins_num = nets[1].ins_linear.weight.shape[0] - 1
    out = M.extract_mesh(nets[1], nets[0], T, grid_dim=a.grid_dim, near=a.near, far=a.far, N_samples=a.N_samples,
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
    print(json.dumps({"vertices": int(out["vertices"].shape[0]), "triangles": int(out["triangles"].shape[0]),
                      "clean_vertices": int(out["clean_vertices"].shape[0]), "clean_triangles": int(out["clean_triangles"].shape[0]),
                      "files": [a.name + ".ply", "color_" + a.name + ".ply"]}))


if __name__ == "__main__":
    main()
