#!/usr/bin/env python
"""Which objects a trained DM-NeRF checkpoint found, and where they are in 3-D (DESIGN.md, "Object inventory").

    python tools/find_objects.py CHECKPOINT.tar (--transform T [--extents X Y Z] | --poses POSES.npy --hwk H W K) [--trim 0]
                                 [--grid-dim 256] [--level 0.45] [--near 4 --far 15] [--out DIR]
                                 [--components {largest,split} [--connectivity {6,26}] [--min-voxels N]]
                                 [--contacts [--down X Y Z]] [--placements L --down X Y Z [--lift N] [--turns K] --out DIR]

CHECKPOINT holds `network_coarse_state_dict` and `network_fine_state_dict`.  The grid is either given (--transform: a 4x4 as
.npy or 16 numbers of text, with --extents, default the original's 1.9 7 7) or found from the cameras (--poses: [N, 4, 4] or
[N, 3, 4] camera-to-world, --hwk: height, width and K as a .npy path or 9 numbers): the scene box of the fine network's solid
points inside the cameras' view, which --out then receives as scene_transform.txt and extents.txt for tools/extract_mesh.py
--extents.  Prints one JSON line: the box used and one entry per object (label, voxels, volume, centre, aabb, obb), all in the
network frame, the frame of the camera poses and of manipulator_eval's transforms.  --components splits each label into
connected components (DESIGN.md, "Connected components"): `largest` reports each object's largest component and adds its
label's component count and discarded voxels; `split` reports every component of at least --min-voxels voxels, with its id.
--contacts adds the touching pairs (DESIGN.md, "Collision checks") of a sweep with the inventory's selection: per index axis its
network-frame direction and one voxel face's area, and per pair of labels (a, b) the faces where a solid point of a has a solid
point of b next to it along +axis, with their area.  --down (network frame) adds to each object `rests_on`: the labels below it
along the index axis closest to that direction, with the faces they share.  --placements L (DESIGN.md, "Object placement") writes
DIR/placements_L.npz: the placement map of label L lowered along --down (raised by --lift voxels first) on the keep-all sweep --
drop, support and contacts [U, V], offset_lo, axis, sign, horizontal, centre (index space), runs and points -- and names it in
the JSON line's `placements`.  --turns K (DESIGN.md, "Turned placements") maps the object turned about down by 360 k / K degrees
instead: the .npz then holds angles (those mapped, in turn order), unfit and unplaced (the angles that did not fit the grid or
left no point), axis, sign, lift, points_before, and per mapped turn t drop_t, support_t, contacts_t, offset_lo_t, base_t,
centre_t and points_t."""
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
    ap.add_argument("--contacts", action="store_true", help="also report which objects touch")
    ap.add_argument("--down", type=float, nargs=3, default=None, metavar=("X", "Y", "Z"),
                    help="with --contacts: the network-frame down direction; adds rests_on per object")
    ap.add_argument("--placements", type=int, default=None, metavar="L", help="write the placement map of label L (needs --down)")
    ap.add_argument("--lift", type=int, default=None, help="with --placements: voxels the object is raised by first (default 0)")
    ap.add_argument("--turns", type=int, default=None, metavar="K",
                    help="with --placements: also the maps of the object turned about down by 360 k / K degrees (default 1)")
    ap.add_argument("--device", default="cuda")
    a = ap.parse_args(argv)
    if a.down is not None and not (a.contacts or a.placements is not None):
        ap.error("--down needs --contacts or --placements")
    if a.placements is not None:
        if a.down is None or a.out is None:
            ap.error("--placements needs --down and --out")
        if not 0 <= a.placements <= 127:
            ap.error("--placements: label %d outside [0, 127]" % a.placements)
        if a.lift is not None and a.lift < 0:
            ap.error("--lift must be >= 0")
        if a.turns is not None and a.turns < 1:
            ap.error("--turns must be >= 1")
        a.turns = a.turns or 1
    elif a.lift is not None or a.turns is not None:
        ap.error("--lift and --turns need --placements")
    if a.down is not None and not any(a.down):
        ap.error("--down must not be 0 0 0")
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


def contacts_json(a, nf, T, ext, objects):
    """--contacts: object_contacts of a sweep keeping every label but the last, as object_inventory sweeps; with --down, each
    entry of `objects` gains rests_on."""
    import torch
    from dmnerf_b200.objects import object_contacts, object_mask, occupancy_objects, supports
    ins_num = int(nf.ins_linear.weight.shape[0]) - 1
    with torch.no_grad():
        occ, labels = occupancy_objects(nf, T, object_mask(ins_num, keep=range(ins_num)), a.grid_dim, tuple(ext), a.near, a.far,
                                        a.N_importance, device=next(nf.parameters()).device)
        c = object_contacts(occ, labels, T, tuple(ext), a.level)
    del occ, labels
    pairs = [{"labels": [int(l1), int(l2)], "axis": int(ax), "faces": int(c["faces"][ax, l1, l2]),
              "area": float(c["faces"][ax, l1, l2] * c["face_area"][ax])} for ax, l1, l2 in zip(*np.nonzero(c["faces"]))]
    if a.down is not None:
        below = supports(c, a.down)
        for e in objects:
            e["rests_on"] = [{"label": k, "faces": n} for k, n in below.get(e["label"], [])]
    return {"contacts": {"axes": c["axes"].tolist(), "face_area": c["face_area"].tolist(), "pairs": pairs}}


def placements_npz(a, nf, T, ext):
    """--placements: placement_map of the label on the keep-all sweep, written to DIR/placements_L.npz -> its file name."""
    import torch
    from dmnerf_b200.objects import object_mask, occupancy_objects, placement_map, turned_placement_maps
    ins_num = int(nf.ins_linear.weight.shape[0]) - 1
    with torch.no_grad():
        occ, labels = occupancy_objects(nf, T, object_mask(ins_num, remove=[]), a.grid_dim, tuple(ext), a.near, a.far, a.N_importance,
                                        device=next(nf.parameters()).device)
        if a.turns == 1:
            m = placement_map(occ, labels, T, a.placements, a.down, a.lift or 0, tuple(ext), a.level)
        else:
            maps, unfit, unplaced = turned_placement_maps(occ, labels, T, a.placements, a.down, a.turns, a.lift or 0, tuple(ext),
                                                          a.level)
    name = "placements_%d.npz" % a.placements
    if a.turns == 1:
        np.savez(os.path.join(a.out, name), drop=m["drop"].cpu().numpy(), support=m["support"].cpu().numpy(),
                 contacts=m["contacts"].cpu().numpy(), offset_lo=np.array(m["offset_lo"]), axis=m["axis"], sign=m["sign"],
                 horizontal=np.array(m["horizontal"]), centre=np.array([float(c) for c in m["centre"]]), runs=m["runs"],
                 points=m["points"], lift=m["lift"])
        return name
    per_turn = {}
    for t, (angle, m) in enumerate(maps):
        per_turn.update({"drop_%d" % t: m["drop"].cpu().numpy(), "support_%d" % t: m["support"].cpu().numpy(),
                         "contacts_%d" % t: m["contacts"].cpu().numpy(), "offset_lo_%d" % t: np.array(m["offset_lo"]),
                         "base_%d" % t: m["base"], "centre_%d" % t: np.array([float(c) for c in m["centre"]]),
                         "points_%d" % t: m["points"]})
    first = maps[0][1] if maps else None
    np.savez(os.path.join(a.out, name), angles=np.array([angle for angle, _ in maps], dtype=np.float64),
             unfit=np.array(unfit, dtype=np.float64), unplaced=np.array(unplaced, dtype=np.float64),
             axis=-1 if first is None else first["axis"], sign=0 if first is None else first["sign"], lift=a.lift or 0,
             points_before=0 if first is None else first["points_before"], **per_turn)
    return name


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
    out = {"objects": [_json(e) for e in inv]}
    if a.contacts:
        out.update(contacts_json(a, nf, T, ext, out["objects"]))
    files = []
    if a.placements is not None:
        os.makedirs(a.out, exist_ok=True)
        out["placements"] = placements_npz(a, nf, T, ext)
        files.append(out["placements"])
    if a.out is not None and a.poses is not None:
        os.makedirs(a.out, exist_ok=True)
        np.savetxt(os.path.join(a.out, "scene_transform.txt"), T, fmt="%.17g")
        np.savetxt(os.path.join(a.out, "extents.txt"), np.asarray(ext).reshape(1, 3), fmt="%.17g")
        files += ["scene_transform.txt", "extents.txt"]
    print(json.dumps({"scene_transform": np.asarray(T).tolist(), "extents": np.asarray(ext).tolist(), "trim": a.trim,
                      **out, "files": files}))


if __name__ == "__main__":
    main()
