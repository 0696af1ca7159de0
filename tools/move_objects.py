#!/usr/bin/env python
"""Move one piece of an object of a trained DM-NeRF checkpoint and render the edited frame (DESIGN.md, "Moving pieces").

    python tools/move_objects.py CHECKPOINT.tar --pose POSE.npy --hwk H W K (--move-label L | --move-piece ID)
           --mode {translation,rotation,scale,multi} [--distance -0.25 --yaw 90 --scale 1.2] [--rest keep|drop]
           --transform T [--extents X Y Z] [--grid-dim 256] [--level 0.45] [--connectivity {6,26}] [--dilate 1] --out DIR
           [--near 4 --far 15 --N-samples 64 --N-importance 128 --N-test 4096] [--mesh [--min-cluster 400]]

CHECKPOINT holds `network_coarse_state_dict` and `network_fine_state_dict`.  POSE.npy holds the camera-to-world pose [4, 4] (or
[3, 4]; of several [N, 4, 4] the first is used).  K is the 3x3 intrinsics, as a .npy file or as 9 numbers.

One labelled occupancy sweep of the fine network over the grid of --transform / --extents / --grid-dim (every label but the last,
as tools/find_objects.py), split at --level into --connectivity-connected pieces, gives the piece: --move-piece takes that
component (the `component` ids of tools/find_objects.py --components split with the same sweep arguments), --move-label the
label's largest one.  The edit turns or shifts the piece about its own centre (manipulation_transform, the original's
generate_poses_eval), moves only that piece (its region grown by --dilate voxels) and keeps (--rest keep) or removes (--rest drop)
the rest of its label: `--move-label L --rest drop` moves object L without its floaters.

Writes DIR/rgb.png, DIR/instance.png (the arg-max label of the edited instance map; label k gets colour k of a fixed seeded
palette, as tools/render_objects.py) and DIR/transform.json (the transformation dict, the moved label, piece and centre), and
prints one JSON line.  --mesh also writes DIR/edited.ply (the marching-cubes mesh of the edited scene, scene space) and
DIR/color_edited.ply (the cleaned mesh, every vertex in its label's colour of instance.png) of the same edit: the same piece,
rest and transformation, applied per grid point to the labelled sweep (DESIGN.md, "Meshing an edited scene")."""
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
    which = ap.add_mutually_exclusive_group(required=True)
    which.add_argument("--move-label", type=int, metavar="L", help="move the largest piece of object label L")
    which.add_argument("--move-piece", type=int, metavar="ID", help="move this piece (a component id of the sweep)")
    ap.add_argument("--mode", required=True, choices=("translation", "rotation", "scale", "multi"))
    ap.add_argument("--distance", type=float, default=-0.25, help="translation along y")
    ap.add_argument("--yaw", type=float, default=90.0, help="rotation about z, degrees")
    ap.add_argument("--scale", type=float, default=1.2)
    ap.add_argument("--rest", choices=("keep", "drop"), default="keep", help="the rest of the moved label: kept or removed")
    ap.add_argument("--transform", required=True, help="4x4 scene transform of the sweep grid (.npy or text)")
    ap.add_argument("--extents", type=float, nargs=3, default=[1.9, 7.0, 7.0], metavar=("X", "Y", "Z"))
    ap.add_argument("--grid-dim", type=int, default=256)
    ap.add_argument("--level", type=float, default=0.45)
    ap.add_argument("--connectivity", type=int, choices=(6, 26), default=26)
    ap.add_argument("--dilate", type=int, default=1, help="voxels the moved piece's region is grown by")
    ap.add_argument("--out", required=True)
    ap.add_argument("--near", type=float, default=4.0)
    ap.add_argument("--far", type=float, default=15.0)
    ap.add_argument("--N-samples", type=int, default=64)
    ap.add_argument("--N-importance", type=int, default=128)
    ap.add_argument("--N-test", type=int, default=4096, help="rays per edit call")
    ap.add_argument("--device", default="cuda")
    ap.add_argument("--mesh", action="store_true", help="also write edited.ply and color_edited.ply of the edit")
    ap.add_argument("--min-cluster", type=int, default=400, help="--mesh: smallest triangle cluster kept in color_edited.ply")
    a = ap.parse_args(argv)
    if a.dilate < 0:
        ap.error("--dilate must be >= 0")
    if len(a.hwk) not in (3, 11):
        ap.error("--hwk takes H W and K as a .npy path or as 9 numbers")
    a.H, a.W = int(a.hwk[0]), int(a.hwk[1])
    a.K = (np.load(a.hwk[2]) if len(a.hwk) == 3 else np.array([float(v) for v in a.hwk[2:]])).astype(np.float32).reshape(3, 3)
    return a


def choose_piece(a, model_fine, T, ext):
    """The sweep, its components and the moved piece -> (component id, its label, its centre, its Region)."""
    import torch
    from dmnerf_b200.objects import (component_region, inventory_from_grid, largest_components, object_components, object_mask,
                                     occupancy_objects)
    ins_num = int(model_fine.ins_linear.weight.shape[0]) - 1
    with torch.no_grad():
        occ, labels = occupancy_objects(model_fine, T, object_mask(ins_num, keep=range(ins_num)), a.grid_dim, ext, a.near, a.far,
                                        a.N_importance, device=next(model_fine.parameters()).device)
        cc = object_components(occ, labels, a.level, a.connectivity)
        if a.move_piece is not None:
            piece = int(a.move_piece)
            if not 0 <= piece < len(cc["label"]):
                raise SystemExit("move_objects: piece %d does not exist (the sweep has %d pieces)" % (piece, len(cc["label"])))
        else:
            best = largest_components(cc["label"], cc["voxels"])
            if a.move_label not in best or a.move_label >= ins_num:
                raise SystemExit("move_objects: object label %d has no piece in the sweep" % a.move_label)
            piece = best[a.move_label]
        label = int(cc["label"][piece])
        inv = inventory_from_grid(occ, labels, T, ext, a.level, objects=[label], components="split",
                                  connectivity=a.connectivity)
    del occ, labels
    centre = next(e["centre"] for e in inv if e["component"] == piece)
    region = component_region(cc, [piece], T, ext, dilate=a.dilate, connectivity=a.connectivity)
    return piece, label, np.asarray(centre, dtype=np.float64), region


def main(argv=None):
    a = parse(argv)
    import torch
    from dmnerf_b200 import mesh as M
    from dmnerf_b200.embedder import get_embedder
    from dmnerf_b200.manipulator import manipulate_frame, rigid_rays
    from dmnerf_b200.mesh import argmax_rows
    from dmnerf_b200.objects import manipulation_transform
    from dmnerf_b200.testing import model_from_weights
    from dmnerf_b200.tester import colorize, pred_label_lut, write_png
    ck = torch.load(a.checkpoint, map_location="cpu")
    nets = [model_from_weights({k: v.float().numpy() for k, v in ck[key].items()}, a.device)
            for key in ("network_coarse_state_dict", "network_fine_state_dict")]
    ins_num = int(nets[1].ins_linear.weight.shape[0]) - 1
    pose = np.load(a.pose).astype(np.float32)
    pose = pose[0] if pose.ndim == 3 else pose
    c2w = np.eye(4, dtype=np.float32)
    c2w[:pose.shape[0]] = pose[:4]
    T = np.load(a.transform) if a.transform.endswith(".npy") else np.loadtxt(a.transform)
    T, ext = M.check_transform(np.asarray(T, dtype=np.float64).reshape(4, 4)), tuple(a.extents)
    piece, label, centre, region = choose_piece(a, nets[1], T, ext)
    trans = manipulation_transform(centre, a.mode, distance=a.distance, yaw=a.yaw, scale=a.scale)
    dev = next(nets[1].parameters()).device
    pose_t = torch.from_numpy(c2w).to(dev)
    tar_o, tar_d = rigid_rays(a.H, a.W, a.K, trans["transformations"][0]["transformation"], pose_t)
    args = types.SimpleNamespace(N_test=a.N_test, N_samples=a.N_samples, N_importance=a.N_importance, near=a.near, far=a.far,
                                 target_labels=[label])
    pe, _ = get_embedder(10)
    ve, _ = get_embedder(4)
    rgb, ins, _, _ = manipulate_frame(a.H, a.W, a.K, pose_t, tar_o[None], tar_d[None], pe, ve, nets[0], nets[1], args,
                                      pieces=[region], rest=a.rest)
    os.makedirs(a.out, exist_ok=True)
    write_png(os.path.join(a.out, "rgb.png"), (255 * torch.clamp(rgb, 0, 1)).to(torch.uint8).reshape(a.H, a.W, 3).cpu().numpy())
    ins_rgbs = np.random.default_rng(0).integers(0, 256, (ins_num + 1, 3))
    lut = pred_label_lut({str(k): k for k in range(ins_num + 1)}, ins_rgbs, {str(k): k for k in range(ins_num + 1)},
                         ins_num + 1)[:, ::-1]
    write_png(os.path.join(a.out, "instance.png"), colorize(argmax_rows(ins).reshape(a.H, a.W), lut).cpu().numpy())
    record = {"transformations": trans["transformations"], "label": label, "piece": piece, "centre": centre.tolist(),
              "rest": a.rest}
    if a.mesh:
        from dmnerf_b200.objects import edited_mesh
        m = edited_mesh(nets[1], T, [(label, trans["transformations"][0]["transformation"])], a.grid_dim, ext, a.level, a.near,
                        a.far, a.N_importance, pieces=[region], rest=a.rest, min_cluster=a.min_cluster)
        M.write_ply(os.path.join(a.out, "edited.ply"), m["vertices"], m["triangles"])
        lab = m["labels"].cpu().numpy()
        colors = np.where((lab >= 0)[:, None], lut[np.clip(lab, 0, ins_num)], 0).astype(np.uint8)   # instance.png's colours
        M.write_ply(os.path.join(a.out, "color_edited.ply"), m["clean_vertices"], m["clean_triangles"], colors)
        record["mesh"] = {"vertices": int(m["vertices"].shape[0]), "triangles": int(m["triangles"].shape[0]),
                          "clean_vertices": int(m["clean_vertices"].shape[0]), "clean_triangles": int(m["clean_triangles"].shape[0])}
    with open(os.path.join(a.out, "transform.json"), "w") as fh:
        json.dump(record, fh, indent=1)
    print(json.dumps(dict(record, files=sorted(os.listdir(a.out)))))


if __name__ == "__main__":
    main()
