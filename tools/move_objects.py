#!/usr/bin/env python
"""Move one piece of an object of a trained DM-NeRF checkpoint and render the edited frame (DESIGN.md, "Moving pieces").

    python tools/move_objects.py CHECKPOINT.tar --pose POSE.npy --hwk H W K
           (--move-label L | --move-piece ID | --pick X Y | --arrange SPEC.json)
           (--mode {translation,rotation,scale,multi} [--distance -0.25 --yaw 90 --scale 1.2]
            | --place-at X Y Z --down X Y Z [--on L ...] [--lift N] [--any-stability] [--turns K]) [--rest keep|drop]
           --transform T [--extents X Y Z] [--grid-dim 256] [--level 0.45] [--connectivity {6,26}] [--dilate 1] --out DIR
           [--near 4 --far 15 --N-samples 64 --N-importance 128 --N-test 4096] [--mesh [--min-cluster 400]]
           [--check] [--until-contact [--step S] [--tolerance N]] [--preview] [--render {exchanger,samples,none}]

CHECKPOINT holds `network_coarse_state_dict` and `network_fine_state_dict`.  POSE.npy holds the camera-to-world pose [4, 4] (or
[3, 4]; of several [N, 4, 4] the first is used).  K is the 3x3 intrinsics, as a .npy file or as 9 numbers.

One labelled occupancy sweep of the fine network over the grid of --transform / --extents / --grid-dim (every label but the last,
as tools/find_objects.py), split at --level into --connectivity-connected pieces, gives the piece: --move-piece takes that
component (the `component` ids of tools/find_objects.py --components split with the same sweep arguments), --move-label the
label's largest one.  The edit turns or shifts the piece about its own centre (manipulation_transform, the original's
generate_poses_eval), moves only that piece (its region grown by --dilate voxels) and keeps (--rest keep) or removes (--rest drop)
the rest of its label: `--move-label L --rest drop` moves object L without its floaters.  --pick X Y takes the piece under
column X, row Y of --pose's view: the pixel's ray (get_rays_at) cast through the same sweep (cast_grid, DESIGN.md, "Viewing the
labelled grid"); the label, piece and network-frame point it hits are printed and recorded as pick.

Writes DIR/rgb.png, DIR/instance.png (the arg-max label of the edited instance map; label k gets colour k of a fixed seeded
palette, as tools/render_objects.py) and DIR/transform.json (the transformation dict, the moved label, piece and centre), and
prints one JSON line.  --mesh also writes DIR/edited.ply (the marching-cubes mesh of the edited scene, scene space) and
DIR/color_edited.ply (the cleaned mesh, every vertex in its label's colour of instance.png) of the same edit: the same piece,
rest and transformation, applied per grid point to the labelled sweep (DESIGN.md, "Meshing an edited scene").

Collision checks (DESIGN.md, "Collision checks") read one keep-all labelled sweep, the one the edited mesh starts from:
--check adds `overlap` (per label, the solid voxels of other objects the moved piece lands on, and their volume) and `landed`
(the voxels it occupies after the move) to transform.json and the JSON line.  --until-contact (--mode translation only) slides
the piece the way --distance moves it, by at most |--distance| in steps of --step (default one grid spacing), and stops before
the first step that overlaps by more than --tolerance voxels; the distance found replaces --distance in the transformation that
is rendered and meshed, and the record gains slide {requested, found, contact}.

Placement (DESIGN.md, "Object placement"): --place-at chooses the move instead of --mode.  The piece is lowered along the index
axis closest to --down (network frame), after being raised by --lift voxels, at every horizontal offset of the keep-all sweep;
of the offsets where it rests on an object (of a label among --on, when given), the one whose centre of mass lands nearest to
the network-frame point --place-at across the down axis, and stands (its centre over the hull of its support; --any-stability:
the nearest, standing or not), is rendered and meshed as --until-contact's is.  The record gains place {offset, drop, support,
stable, contacts}.  --turns K (DESIGN.md, "Turned placements") also turns the piece about down by 360 k / K degrees and picks the
nearest placement over every turn that fits the grid; the record's place gains turn, the angle in degrees of the one chosen.

Arranging (DESIGN.md, "Arranging objects"): --arrange SPEC.json --down X Y Z replaces --move-label / --move-piece and places
several objects one after another, each in the scene the earlier placements leave (objects.arrange_objects).  SPEC is a list of
{"label": L | "piece": ID, "near": [x, y, z], "on": [...], "turns": K, "rest": "keep" | "drop", "any_stability": bool}: "label"
moves the label's largest piece and "piece" that component, each with its region grown by --dilate voxels, as the single-move
flags do.  The frame is rendered with every placed move (manipulate_frame), --mesh meshes the same moves (edited_mesh), and the
record gains arrange: per item label, placed, reason, offset, drop, support, stable and turn, and each placed move's overwritten
(the solid voxels of the scene left before it that it landed on, per label).

Rendering (--render): `exchanger` (the default) renders the frame with manipulate_frame, the original's exchanger, which renders
the scene again along every move.  `samples` renders the same moves, pieces and rest with render_frame(moves=) (DESIGN.md,
"Rendering moved objects"): the edited sweep's rule applied per render sample, with the default boxes of the keep-all sweep, so
that the frame and --mesh show the same edit.  The record gains render and evaluated (the targets the moved render evaluated in
its coarse and fine passes; null for the exchanger).  `none` renders no frame and meshes nothing: with --preview, the look at an
edit costs a grid edit and a voxel walk per pixel instead of a network render.

Previews (--preview; DESIGN.md, "Viewing the labelled grid"): before the frame is rendered, the keep-all sweep is cast from --pose
(grid_view): DIR/preview.png shows the unedited grid and DIR/preview_edited.png the edited_grid of the same moves (or the
arrangement), in instance.png's colours shaded by the angle between surface and ray, DIR/preview_rgb.png the network's colour
at the unedited grid's hits (one query per pixel) and DIR/preview_edited_rgb.png the edited grid in the edit's network colour:
each hit traced to the move that placed it and coloured from the network at that move's source (grid_view(moves=, source=);
DESIGN.md, "Colouring an edited view"), for every edit the tool builds.

Deforming (--twist DEG, --bend D --bend-dir X Y Z, --taper S, with --up X Y Z and --knots K; DESIGN.md, "Deforming objects"):
the piece is twisted, bent and tapered before its move, about its inventory centre, over its extent along --up in the sweep; the
twist (0 to DEG) and taper (1 to S) are linear in height and the bend (0 to D) quadratic.  They need --render samples, work with
--mesh and --check, and the record gains deformation."""
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
    which.add_argument("--pick", type=int, nargs=2, metavar=("X", "Y"), help="move the piece under column X, row Y of --pose's view")
    which.add_argument("--arrange", metavar="SPEC.json", help="place several pieces one after another (a JSON list of items)")
    ap.add_argument("--mode", choices=("translation", "rotation", "scale", "multi"))
    ap.add_argument("--distance", type=float, default=None, help="translation along y (default -0.25)")
    ap.add_argument("--yaw", type=float, default=None, help="rotation about z, degrees (default 90)")
    ap.add_argument("--scale", type=float, default=None, help="(default 1.2)")
    ap.add_argument("--place-at", type=float, nargs=3, default=None, metavar=("X", "Y", "Z"),
                    help="place the piece where it rests nearest to this network-frame point (replaces --mode)")
    ap.add_argument("--down", type=float, nargs=3, default=None, metavar=("X", "Y", "Z"), help="--place-at: network-frame down")
    ap.add_argument("--on", type=int, nargs="+", default=None, metavar="L", help="--place-at: rest on one of these labels")
    ap.add_argument("--lift", type=int, default=None, help="--place-at: voxels the piece is raised by first (default 0)")
    ap.add_argument("--any-stability", action="store_true", help="--place-at: take the nearest resting offset, stable or not")
    ap.add_argument("--turns", type=int, default=None, metavar="K",
                    help="--place-at: also turn the piece about down by 360 k / K degrees, k = 0 .. K - 1 (default 1: unturned)")
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
    ap.add_argument("--check", action="store_true", help="report the overlap of the move with the other objects")
    ap.add_argument("--until-contact", action="store_true", help="translation: slide until just before contact")
    ap.add_argument("--step", type=float, default=None, help="--until-contact: the slide's step (default: one grid spacing)")
    ap.add_argument("--tolerance", type=int, default=0, help="--until-contact: overlapping voxels tolerated")
    ap.add_argument("--render", choices=("exchanger", "samples", "none"), default="exchanger",
                    help="render the frame with the exchanger (manipulate_frame), per sample (render_frame(moves=)) or not at all")
    ap.add_argument("--preview", action="store_true",
                    help="write preview.png, preview_edited.png, preview_rgb.png and preview_edited_rgb.png: the sweep cast "
                         "from --pose, before and after, in label and network colours")
    ap.add_argument("--copy", action="store_true", help="copy the piece instead of moving it: the source stays (needs --render samples)")
    ap.add_argument("--with", dest="with_labels", type=int, nargs="+", default=None, metavar="L",
                    help="move these labels together with the piece's label, as one body (needs --render samples)")
    ap.add_argument("--carry", action="store_true",
                    help="also move what rests on the piece's label, transitively (carried_labels; needs --down and --render samples)")
    ap.add_argument("--twist", type=float, default=None, metavar="DEG",
                    help="twist the piece about --up, 0 at its bottom to DEG at its top (needs --render samples)")
    ap.add_argument("--bend", type=float, default=None, metavar="D",
                    help="bend the piece: its top shifts by D along --bend-dir, quadratic in height (needs --render samples)")
    ap.add_argument("--bend-dir", type=float, nargs=3, default=None, metavar=("X", "Y", "Z"), help="--bend: the horizontal direction")
    ap.add_argument("--taper", type=float, default=None, metavar="S",
                    help="taper the piece: horizontal scale 1 at its bottom to S at its top (needs --render samples)")
    ap.add_argument("--up", type=float, nargs=3, default=None, metavar=("X", "Y", "Z"),
                    help="--twist / --bend / --taper: the network-frame up axis of the deformation")
    ap.add_argument("--knots", type=int, default=33, help="--twist / --bend / --taper: knots of the deformation's table")
    a = ap.parse_args(argv)
    a.deformed = a.twist is not None or a.bend is not None or a.taper is not None
    if a.render == "none":
        if not a.preview:
            ap.error("--render none needs --preview: there would be nothing to look at")
        if a.mesh:
            ap.error("--render none stops after the preview: drop --mesh")
    if a.deformed:
        if a.render == "exchanger":
            ap.error("--twist, --bend and --taper need --render samples: the exchanger renders rigid moves only")
        for flag, given in (("--arrange", a.arrange is not None), ("--place-at", a.place_at is not None),
                            ("--until-contact", a.until_contact)):
            if given:
                ap.error("--twist, --bend and --taper cannot be combined with %s: placement and the slide are rigid" % flag)
        if a.up is None or not any(a.up):
            ap.error("--twist, --bend and --taper need --up X Y Z, not 0 0 0")
        if a.bend is not None and (a.bend_dir is None or not any(a.bend_dir)):
            ap.error("--bend needs --bend-dir X Y Z, not 0 0 0")
        if not 2 <= a.knots <= 64:
            ap.error("deformation: n_knots %d is not 0 and outside [2, 64]" % a.knots)
        if a.taper is not None and not a.taper > 0:
            ap.error("deformation: taper must be > 0")
    elif a.up is not None or a.bend_dir is not None:
        ap.error("--up and --bend-dir need --twist, --bend or --taper")
    a.grouped = a.with_labels is not None or a.carry
    if a.grouped:
        if a.arrange is not None:
            ap.error('--with and --carry are per item with --arrange: give the items "group": [labels]')
        if a.render == "exchanger":
            ap.error("--with and --carry need --render samples: the exchanger renders one label per move")
        if a.carry and (a.down is None or not any(a.down)):
            ap.error("--carry needs --down X Y Z, not 0 0 0: what rests on the object is found along it")
        if a.until_contact:
            ap.error("--with and --carry cannot be combined with --until-contact: the slide moves one label")
    if a.copy:
        if a.render == "exchanger":
            ap.error("--copy needs --render samples: the exchanger renders moves only")
        if a.rest == "drop":
            ap.error("--copy cannot drop the rest of the label: a copy vacates nothing")
        if a.until_contact:
            ap.error("--copy cannot be combined with --until-contact: a copy starts inside its source")
    if a.arrange is not None:
        for flag, given in (("--place-at", a.place_at is not None), ("--mode", a.mode is not None),
                            ("--until-contact", a.until_contact), ("--distance", a.distance is not None), ("--yaw", a.yaw is not None),
                            ("--scale", a.scale is not None), ("--turns", a.turns is not None), ("--check", a.check)):
            if given:
                ap.error("--arrange cannot be combined with %s (each item gives its own placement; the record reports what "
                         "each placed move overwrote)" % flag)
        if a.down is None or not any(a.down):
            ap.error("--arrange needs --down X Y Z, not 0 0 0")
        if a.on is not None or a.lift is not None or a.any_stability:
            ap.error("--on, --lift and --any-stability are per item with --arrange")
        if a.copy:
            ap.error('--copy is per item with --arrange: give the items "copy": true')
        a.lift, a.turns = 0, 1
    elif a.place_at is not None:
        for flag, given in (("--mode", a.mode is not None), ("--until-contact", a.until_contact), ("--distance", a.distance is not None),
                            ("--yaw", a.yaw is not None), ("--scale", a.scale is not None)):
            if given:
                ap.error("--place-at replaces %s" % flag)
        if a.down is None or not any(a.down):
            ap.error("--place-at needs --down X Y Z, not 0 0 0")
        if a.lift is not None and a.lift < 0:
            ap.error("--lift must be >= 0")
        if a.turns is not None and a.turns < 1:
            ap.error("--turns must be >= 1")
        a.lift = a.lift or 0
        a.turns = a.turns or 1
    else:
        if a.mode is None:
            ap.error("give --mode or --place-at")
        if (a.down is not None and not a.carry) or a.on is not None or a.lift is not None or a.any_stability or a.turns is not None:
            ap.error("--down, --on, --lift, --any-stability and --turns need --place-at (--down also serves --carry)")
        a.distance = -0.25 if a.distance is None else a.distance
        a.yaw = 90.0 if a.yaw is None else a.yaw
        a.scale = 1.2 if a.scale is None else a.scale
    if a.until_contact:
        if a.mode != "translation":
            ap.error("--until-contact needs --mode translation")
        if a.distance == 0:
            ap.error("--until-contact needs a non-zero --distance (its sign gives the direction)")
        if a.step is not None and not a.step > 0:
            ap.error("--step must be > 0")
        if a.tolerance < 0:
            ap.error("--tolerance must be >= 0")
    elif a.step is not None or a.tolerance != 0:
        ap.error("--step and --tolerance need --until-contact")
    if a.dilate < 0:
        ap.error("--dilate must be >= 0")
    if len(a.hwk) not in (3, 11):
        ap.error("--hwk takes H W and K as a .npy path or as 9 numbers")
    a.H, a.W = int(a.hwk[0]), int(a.hwk[1])
    a.K = (np.load(a.hwk[2]) if len(a.hwk) == 3 else np.array([float(v) for v in a.hwk[2:]])).astype(np.float32).reshape(3, 3)
    if a.pick is not None and not (0 <= a.pick[0] < a.W and 0 <= a.pick[1] < a.H):
        ap.error("--pick %d %d is outside the %d x %d view" % (a.pick[0], a.pick[1], a.W, a.H))
    a.picked = None
    return a


ITEM_KEYS = ("label", "piece", "near", "on", "turns", "rest", "any_stability", "copy", "group")


def read_spec(path):
    """--arrange's SPEC -> [item dict]; SystemExit for a malformed one."""
    with open(path) as fh:
        spec = json.load(fh)
    if not isinstance(spec, list) or not spec:
        raise SystemExit("move_objects: %s must hold a non-empty JSON list of items" % path)
    for i, it in enumerate(spec):
        if not isinstance(it, dict) or set(it) - set(ITEM_KEYS) or ("label" in it) == ("piece" in it) or "near" not in it:
            raise SystemExit("move_objects: item %d of %s needs exactly one of label / piece, near, and only the keys %s"
                             % (i, path, ", ".join(ITEM_KEYS)))
        if not isinstance(it.get("copy", False), bool):
            raise SystemExit("move_objects: item %d of %s: copy must be true or false" % (i, path))
        g = it.get("group")
        if g is not None and (not isinstance(g, list) or not all(isinstance(k, int) and not isinstance(k, bool) for k in g)):
            raise SystemExit("move_objects: item %d of %s: group must be a list of labels" % (i, path))
        if g is not None and "label" in it and it["label"] not in g:
            raise SystemExit("move_objects: item %d of %s: the group %s does not hold the item's label %d" % (i, path, g, it["label"]))
    return spec


def choose_pieces(a, model_fine, T, ext, spec):
    """choose_piece for every item of --arrange -> [(component id, label, Region)] (one sweep and one split)."""
    import torch
    from dmnerf_b200.objects import component_region, largest_components, object_components, object_mask, occupancy_objects
    ins_num = int(model_fine.ins_linear.weight.shape[0]) - 1
    with torch.no_grad():
        occ, labels = occupancy_objects(model_fine, T, object_mask(ins_num, keep=range(ins_num)), a.grid_dim, ext, a.near, a.far,
                                        a.N_importance, device=next(model_fine.parameters()).device)
        cc = object_components(occ, labels, a.level, a.connectivity)
    del occ, labels
    best = largest_components(cc["label"], cc["voxels"])
    out = []
    for it in spec:
        if "piece" in it:
            piece = int(it["piece"])
            if not 0 <= piece < len(cc["label"]):
                raise SystemExit("move_objects: piece %d does not exist (the sweep has %d pieces)" % (piece, len(cc["label"])))
        else:
            if int(it["label"]) not in best or int(it["label"]) >= ins_num:
                raise SystemExit("move_objects: object label %d has no piece in the sweep" % int(it["label"]))
            piece = best[int(it["label"])]
        out.append((piece, int(cc["label"][piece]), component_region(cc, [piece], T, ext, dilate=a.dilate, connectivity=a.connectivity)))
    return out


def arrange_pieces(a, occ, labels, T, ext, spec, chosen):
    """--arrange: arrange_objects for the items -> (moves, regions, rests, the record's arrange)."""
    from dmnerf_b200.objects import arrange_objects
    items = []
    for i, (it, (_, label, region)) in enumerate(zip(spec, chosen)):
        if it.get("group") is not None and label not in it["group"]:        # a piece item: its label is known from the sweep
            raise SystemExit("move_objects: item %d: the group %s does not hold the label %d of its piece" % (i, it["group"], label))
        items.append({"label": label, "near": it["near"], "on": it.get("on"), "piece": region, "rest": it.get("rest", "keep"),
                      "turns": it.get("turns"), "stable": not it.get("any_stability", False), "copy": it.get("copy", False),
                      "group": it.get("group")})
    r = arrange_objects(occ, labels, T, items, a.down, ext, a.level)
    rec, report = [], iter(r["report"])
    for it, (piece, label, _), res in zip(spec, chosen, r["items"]):
        p = res["placement"]
        entry = {"label": label, "piece": piece, "placed": p is not None, "reason": res.get("reason"),
                 "offset": None if p is None else list(p["offset"]), "drop": None if p is None else p["drop"],
                 "support": None if p is None else p["support"], "stable": None if p is None else p["stable"],
                 "turn": res.get("turn"), "copy": bool(it.get("copy", False)),
                 "group": None if it.get("group") is None else sorted(set(it["group"]))}
        if p is not None:
            entry["overwritten"] = {str(k): v for k, v in next(report)["overwritten"].items()}
        rec.append(entry)
    return r["moves"], r["pieces"], r["rest"], r["copies"], r["groups"], rec, (r["occ"], r["labels"])


def pick_piece(a, occ, labels, T, ext, cc, pose_t):
    """--pick: the piece under the pixel, from its ray cast through the sweep -> (component id, {label, piece, pixel, point});
    exits on a miss."""
    from dmnerf_b200.helpers import get_rays_at
    from dmnerf_b200.objects import cast_grid
    x, y = a.pick
    o, d = get_rays_at(a.H, a.W, a.K, pose_t, [y * a.W + x])
    c = cast_grid(occ, labels, T, o, d, a.near, a.far, ext, a.level, components=cc, normals=False)
    piece = int(c["piece"][0])
    if piece < 0:
        raise SystemExit("move_objects: --pick %d %d: the pixel's ray hits no solid voxel of the sweep between near %g and far %g"
                         % (x, y, a.near, a.far))
    rec = {"pixel": [x, y], "label": int(c["label"][0]), "piece": piece, "point": c["point"][0].tolist()}
    print("move_objects: picked label %d, piece %d at (%.4f, %.4f, %.4f)" % (rec["label"], piece, *rec["point"]))
    return piece, rec


def choose_piece(a, model_fine, T, ext, pose_t=None):
    """The sweep, its components and the moved piece -> (component id, its label, its centre, its Region).  --pick (pose_t: the
    pose on the device) also leaves the pick's record in a.picked."""
    import torch
    from dmnerf_b200.objects import (component_region, inventory_from_grid, largest_components, object_components, object_mask,
                                     occupancy_objects)
    ins_num = int(model_fine.ins_linear.weight.shape[0]) - 1
    with torch.no_grad():
        occ, labels = occupancy_objects(model_fine, T, object_mask(ins_num, keep=range(ins_num)), a.grid_dim, ext, a.near, a.far,
                                        a.N_importance, device=next(model_fine.parameters()).device)
        cc = object_components(occ, labels, a.level, a.connectivity)
        if a.pick is not None:
            piece, a.picked = pick_piece(a, occ, labels, T, ext, cc, pose_t)
        elif a.move_piece is not None:
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


def slide_translation(a, occ, labels, T, ext, label, region):
    """--until-contact: the slide of the piece along the way --distance moves it (manipulation_transform's translation shifts
    the object by -distance along y) -> {requested, found, contact}; found is None when the piece overlaps where it stands."""
    from dmnerf_b200.objects import slide_until_contact
    r = slide_until_contact(occ, labels, T, label, (0.0, -float(np.sign(a.distance)), 0.0), abs(a.distance), step=a.step,
                            tolerance=a.tolerance, extents=ext, level=a.level, piece=region, rest=a.rest)
    contact = None if r["contact"] is None else {"distance": r["contact"]["distance"],
                                                 "overlap": {str(k): v for k, v in r["contact"]["overlap"].items()}}
    return {"requested": a.distance, "found": r["distance"], "contact": contact}


def place_piece(a, occ, labels, T, ext, label, region, group=None):
    """--place-at: place_object for the piece -> {transformation, offset, drop, support, stable, contacts}; exits when no offset
    qualifies."""
    from dmnerf_b200.objects import place_object
    r = place_object(occ, labels, T, label, a.down, a.place_at, on=a.on, stable=not a.any_stability, lift=a.lift, extents=ext,
                     level=a.level, piece=region, rest=a.rest, turns=None if a.turns == 1 else a.turns, copy=a.copy, group=group)
    p = r["placement"]
    if p is None:
        raise SystemExit("move_objects: no placement: %s" % r["reason"])
    out = {"transformation": p["transformation"], "offset": list(p["offset"]), "drop": p["drop"], "support": p["support"],
           "stable": p["stable"], "contacts": [list(c) for c in p["contacts"]]}
    if a.turns != 1:
        out["turn"] = r["turn"]
    return out


def piece_deformation(a, occ, labels, T, ext, label, region, centre):
    """--twist / --bend / --taper: the piece's Deformation about its inventory centre and --up, over the piece's extent along
    --up in the sweep; the twist and taper are linear in height and the bend quadratic."""
    from dmnerf_b200.objects import _region_keeps, deformation, grid_affine
    up = np.asarray(a.up, dtype=np.float64) / np.linalg.norm(a.up)
    mask = (labels == label) & (occ > a.level) & _region_keeps(region, T, occ.shape[0], ext, occ.device)
    A, b = grid_affine(T, occ.shape[0], ext)
    h = (np.argwhere(mask.cpu().numpy()) @ A.T + b - centre) @ up
    h0, h1 = (float(h.min()), float(h.max())) if h.size else (-1.0, 1.0)
    if not h1 > h0:
        h0, h1 = h0 - 1.0, h1 + 1.0
    return deformation(centre, up, h0, h1, a.knots, twist=None if a.twist is None else (lambda s: a.twist * s),
                       bend=None if a.bend is None else (lambda s: a.bend * s * s), bend_dir=a.bend_dir,
                       taper=None if a.taper is None else (lambda s: 1.0 + (a.taper - 1.0) * s))


def write_previews(a, model_fine, occ, labels, T, ext, pose_t, lut, moves, regions, rests, copies, groups, deforms, arranged_grid):
    """--preview: preview.png and preview_rgb.png of the keep-all sweep, preview_edited.png and preview_edited_rgb.png of its
    edited_grid under the moves (or the arranged grid), all cast from --pose (grid_view); the edited colour traces each hit to
    the move that placed it (grid_view(moves=, source=))."""
    import torch
    from dmnerf_b200.objects import edited_grid, grid_view, render_moves
    from dmnerf_b200.tester import write_png
    with torch.no_grad():
        before = grid_view(occ, labels, T, a.H, a.W, a.K, pose_t, a.near, a.far, ext, a.level, lut=lut, model_fine=model_fine)
        if arranged_grid is None:
            e_occ, e_labels, _ = edited_grid(occ, labels, T, moves, ext, a.level, pieces=regions, rest=rests, copies=copies,
                                             groups=groups, deformations=deforms)
        else:
            e_occ, e_labels = arranged_grid
        moved = render_moves(occ, labels, T, moves, ext, a.level, a.near, a.far, a.N_importance, pieces=regions, rest=rests,
                             copies=copies, groups=groups, deformations=deforms)
        after = grid_view(e_occ, e_labels, T, a.H, a.W, a.K, pose_t, a.near, a.far, ext, a.level, lut=lut, model_fine=model_fine,
                          moves=moved, source=(occ, labels))
    to8 = lambda rgb: (255 * torch.clamp(rgb, 0, 1)).to(torch.uint8).cpu().numpy()   # noqa: E731
    write_png(os.path.join(a.out, "preview.png"), before["image"].cpu().numpy())
    write_png(os.path.join(a.out, "preview_edited.png"), after["image"].cpu().numpy())
    write_png(os.path.join(a.out, "preview_rgb.png"), to8(before["rgb"]))
    write_png(os.path.join(a.out, "preview_edited_rgb.png"), to8(after["rgb"]))


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
    slide = place = arranged = None
    dev = next(nets[1].parameters()).device
    pose_t = torch.from_numpy(c2w).to(dev)
    if a.arrange is not None:
        spec = read_spec(a.arrange)
        if any(it.get("copy", False) for it in spec) and a.render == "exchanger":
            raise SystemExit("move_objects: an arrangement with copies needs --render samples: the exchanger renders moves only")
        if any(it.get("group") is not None for it in spec) and a.render == "exchanger":
            raise SystemExit("move_objects: an arrangement with groups needs --render samples: the exchanger renders one label per "
                             "move")
        chosen = choose_pieces(a, nets[1], T, ext, spec)
        piece, label, centre, region = None, None, None, None
    else:
        piece, label, centre, region = choose_piece(a, nets[1], T, ext, pose_t)
    sweep = (a.check or a.until_contact or a.place_at is not None or a.arrange is not None or a.render == "samples" or a.grouped
             or a.preview)
    if sweep:
        from dmnerf_b200.objects import object_mask, occupancy_objects
        with torch.no_grad():
            occ, labels = occupancy_objects(nets[1], T, object_mask(ins_num, remove=[]), a.grid_dim, ext, a.near, a.far,
                                            a.N_importance, device=next(nets[1].parameters()).device)
    group = chain = arranged_grid = None
    if a.grouped:                                      # the piece's label and the labels moved with it
        group = sorted(set(a.with_labels or []) | {label})
        if a.carry:
            from dmnerf_b200.objects import carried_labels
            c = carried_labels(occ, labels, T, label, a.down, ext, a.level)
            group = sorted(set(group) | set(c["group"]))
            chain = {str(k): [b, f] for k, (b, f) in c["chain"].items()}
    if a.until_contact:
        slide = slide_translation(a, occ, labels, T, ext, label, region)
        a.distance = np.sign(a.distance) * (slide["found"] or 0.0)
    if a.arrange is not None:
        moves, regions, rests, copies, groups, arranged, arranged_grid = arrange_pieces(a, occ, labels, T, ext, spec, chosen)
        if not moves:
            raise SystemExit("move_objects: no item was placed: %s" % "; ".join("%d: %s" % (e["label"], e["reason"]) for e in arranged))
        trans = {"transformations": [{"transformation": m, "mode": "placement"} for _, m in moves]}
    elif a.place_at is not None:
        place = place_piece(a, occ, labels, T, ext, label, region, group)
        trans = {"transformations": [{"transformation": place.pop("transformation"), "mode": "placement"}]}
    else:
        trans = manipulation_transform(centre, a.mode, distance=a.distance, yaw=a.yaw, scale=a.scale)
    deforms = None
    if a.arrange is None:
        moves, regions, rests = [(label, trans["transformations"][0]["transformation"])], [region], [a.rest]
        copies, groups = [a.copy], [group]
        if a.deformed:
            deforms = [piece_deformation(a, occ, labels, T, ext, label, region, centre)]
    os.makedirs(a.out, exist_ok=True)
    ins_rgbs = np.random.default_rng(0).integers(0, 256, (ins_num + 1, 3))
    lut = pred_label_lut({str(k): k for k in range(ins_num + 1)}, ins_rgbs, {str(k): k for k in range(ins_num + 1)},
                         ins_num + 1)[:, ::-1]
    if a.preview:
        write_previews(a, nets[1], occ, labels, T, ext, pose_t, lut, moves, regions, rests, copies, groups, deforms, arranged_grid)
    evaluated = None
    if a.render == "samples":
        from dmnerf_b200.objects import render_moves
        from dmnerf_b200.render import render_frame
        moved = render_moves(occ, labels, T, moves, ext, a.level, a.near, a.far, a.N_importance, pieces=regions, rest=rests,
                             copies=copies, groups=groups, deformations=deforms)
        with torch.no_grad():
            fr = render_frame(a.H, a.W, a.K, pose_t, a.near, a.far, nets[0], nets[1], a.N_samples, a.N_importance, keep_all_ins=True,
                              device=dev, moves=moved)
        rgb, ins, evaluated = fr["rgb"].reshape(-1, 3).to(dev), fr["ins"].reshape(a.H * a.W, -1).to(dev), list(fr["evaluated"])
    elif a.render == "exchanger":
        rays = [rigid_rays(a.H, a.W, a.K, m, pose_t) for _, m in moves]
        tar_o, tar_d = torch.stack([o for o, _ in rays]), torch.stack([d for _, d in rays])
        args = types.SimpleNamespace(N_test=a.N_test, N_samples=a.N_samples, N_importance=a.N_importance, near=a.near, far=a.far,
                                     target_labels=[k for k, _ in moves])
        pe, _ = get_embedder(10)
        ve, _ = get_embedder(4)
        rgb, ins, _, _ = manipulate_frame(a.H, a.W, a.K, pose_t, tar_o, tar_d, pe, ve, nets[0], nets[1], args, pieces=regions,
                                          rest=rests)
    if a.render != "none":
        write_png(os.path.join(a.out, "rgb.png"), (255 * torch.clamp(rgb, 0, 1)).to(torch.uint8).reshape(a.H, a.W, 3).cpu().numpy())
        write_png(os.path.join(a.out, "instance.png"), colorize(argmax_rows(ins).reshape(a.H, a.W), lut).cpu().numpy())
    if a.arrange is not None:
        record = {"transformations": trans["transformations"], "labels": [k for k, _ in moves], "rest": rests, "arrange": arranged}
    else:
        record = {"transformations": trans["transformations"], "label": label, "piece": piece, "centre": centre.tolist(),
                  "rest": a.rest}
    record["render"], record["evaluated"] = a.render, evaluated
    if a.picked is not None:
        record["pick"] = a.picked
    if any(copies):
        record["copies"] = copies
    if group is not None:
        record["group"] = group
    if chain is not None:
        record["chain"] = chain
    if deforms is not None:
        record["deformation"] = {"twist": a.twist, "bend": a.bend, "bend_dir": a.bend_dir, "taper": a.taper, "up": a.up,
                                 "knots": a.knots, "h0": deforms[0].h0, "dh": deforms[0].dh}
    if slide is not None:
        record["slide"] = slide
    if place is not None:
        record["place"] = place
    if a.check:
        from dmnerf_b200.objects import move_overlap
        r = move_overlap(occ, labels, T, [(label, trans["transformations"][0]["transformation"])], ext, a.level, pieces=[region],
                         rest=a.rest, copies=a.copy, groups=[group], deformations=deforms)[0]
        record["overlap"] = {"voxels": {str(k): v for k, v in r["overlap"].items()},
                             "volume": {str(k): v for k, v in r["overlap_volume"].items()}}
        record["landed"] = r["landed"]
    if sweep:
        del occ, labels
    if a.mesh:
        from dmnerf_b200.objects import edited_mesh
        m = edited_mesh(nets[1], T, moves, a.grid_dim, ext, a.level, a.near, a.far, a.N_importance, pieces=regions, rest=rests,
                        min_cluster=a.min_cluster, copies=copies, groups=groups, deformations=deforms)
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
