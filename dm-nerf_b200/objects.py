"""Object selection: render or mesh chosen objects of a trained scene (DESIGN.md, "Object selection").

    object_mask(ins_num, keep=None, remove=None)        -> the 4-word mask of kept labels
    render_objects(position_embedder, view_embedder, model_coarse, model_fine, poses, hwk, args, keep=None, remove=None, ...)
                                                        -> isolated / removed views through the frame driver
    object_meshes(model_fine, model_coarse, scene_transform, objects=None, grid_dim=256, level=0.45, ...)
                                                        -> {label: closed mesh of that object}
    object_inventory(model_fine, scene_transform, extents=None, grid_dim=256, level=0.45, trim=0.0, objects=None, ...)
                                                        -> per object: voxels, volume, centre, covariance, aabb, obb (network frame)
    object_components(occ, labels=None, level=0.45, connectivity=26)
                                                        -> the connected components of a labelled grid's solid points
    component_region(cc, ids, scene_transform, ...) / region_from_mask(mask, scene_transform, ...)
                                                        -> a Region: grid bits the renderer reads per sample (render_*(region=))
    region_contains(region, pts)                        -> which points a region keeps, by the render kernels' own test
    Appearance(ins_num, colour=None, density=None), tint(rgb)
                                                        -> per-object colour maps and density scales (render_*(appearance=))
    scene_box(model_fine, poses, hwk, near, far, ...)   -> (scene_transform, extents) of the scene, from the cameras
    manipulation_transform(centre, mode)                -> the transformation dict manipulator_eval takes, about that centre
    edited_sweep(model_fine, scene_transform, moves, ...) / edited_mesh(...)
                                                        -> the labelled sweep / the mesh of a scene with objects moved

Every network sample is labelled argmax(sigmoid(instance logits)) over all ins_num + 1 channels, first maximum winning (the
exchanger's rule); a sample whose label is not kept has alpha = 0 in the composite of both passes, so the coarse weights of the
selected scene drive the importance sampling.  The instance map keeps the network's channels: selection does not re-label it."""
import ctypes as C
import os

import numpy as np
import torch

from . import _lib
from .engine import get_context

MAX_LABELS = 128                     # ins_num + 1 <= 128


def _labels(values, ins_num, what):
    out = []
    for v in values:
        if isinstance(v, (bool, np.bool_)) or int(v) != v:
            raise ValueError("%s: object labels are integers, got %r" % (what, v))
        k = int(v)
        if not 0 <= k <= ins_num:
            raise ValueError("%s: label %d outside [0, %d]" % (what, k, ins_num))
        out.append(k)
    return out


def object_mask(ins_num, keep=None, remove=None):
    """The selection as 4 uint32 words (bit k of word k // 32 = label k is kept), for labels 0 .. ins_num.  Give exactly one of
    keep (the labels to keep; may be empty) or remove (the labels to drop; every other label is kept)."""
    ins_num = int(ins_num)
    if not 1 <= ins_num <= MAX_LABELS - 1:
        raise ValueError("object_mask: ins_num %d outside [1, %d]" % (ins_num, MAX_LABELS - 1))
    if (keep is None) == (remove is None):
        raise ValueError("object_mask: give exactly one of keep= or remove=")
    if keep is not None:
        kept = set(_labels(keep, ins_num, "object_mask"))
    else:
        kept = set(range(ins_num + 1)) - set(_labels(remove, ins_num, "object_mask"))
    words = [0, 0, 0, 0]
    for k in kept:
        words[k >> 5] |= 1 << (k & 31)
    return words


def kept_labels(words):
    """The labels a mask keeps, ascending."""
    return [k for k in range(MAX_LABELS) if (words[k >> 5] >> (k & 31)) & 1]


# ----------------------------------------------------------------------------------------------------------------- views
def _to8b(x):
    return (255 * np.clip(np.asarray(x), 0, 1)).astype(np.uint8)


def render_objects(position_embedder, view_embedder, model_coarse, model_fine, poses, hwk, args, keep=None, remove=None,
                   savedir=None, ins_rgbs=None, color_dict=None, impl=_lib.IMPL_AUTO, region=None, appearance=None):
    """Render every pose (camera-to-world, [4, 4] or [3, 4]) with the selection, deterministically, through the frame driver.
    Reads args.near, args.far, args.N_samples, args.N_importance.  Returns one dict per pose of device maps: rgb [H, W, 3],
    ins [H, W, ins_num], depth [H, W], acc [H, W].
    savedir: writes {i:03d}.png (RGBA, alpha = acc: an isolated object is a cut-out) and instance_{i:03d}.png (the arg-max label
    of the instance map, coloured as render_test colours it: ins_rgbs[color_dict[label]], channels in cv2's order).  Without
    ins_rgbs / color_dict, label k gets colour k of a fixed seeded palette.  impl: the network, as in render_frame.
    region: a Region (region selection, DESIGN.md "Region selection") applied with the label selection; with a region, keep and
    remove may both be left out (every label kept).  Floater cleanup, for example, is the component_region of each object
    label's largest piece (see component_region).
    appearance: an Appearance (object appearance, DESIGN.md "Object appearance") applied to the samples the selection and the
    region keep; with one, keep and remove may both be left out as well."""
    from .render import _check_embedders, render_frame
    from .tester import colorize, pred_label_lut, write_png
    _check_embedders(position_embedder, view_embedder)
    H, W, K = hwk
    H, W = int(H), int(W)
    dev = next(model_fine.parameters()).device
    ins_num = int(model_fine.ins_linear.weight.shape[0]) - 1
    if (region is not None or appearance is not None) and keep is None and remove is None:
        kept = None
    else:
        kept = kept_labels(object_mask(ins_num, keep=keep, remove=remove))
    lut = None
    if savedir is not None:
        os.makedirs(savedir, exist_ok=True)
        if ins_rgbs is None:
            ins_rgbs = np.random.default_rng(0).integers(0, 256, (ins_num + 1, 3))
        if color_dict is None:
            color_dict = {str(k): k for k in range(ins_num + 1)}
        lut = pred_label_lut({str(k): k for k in range(ins_num + 1) if str(k) in color_dict}, ins_rgbs, color_dict,
                             ins_num + 1)[:, ::-1]
    out = []
    with torch.no_grad():
        for i, c2w in enumerate(poses):
            c2w = torch.as_tensor(np.asarray(c2w.cpu() if torch.is_tensor(c2w) else c2w), dtype=torch.float32)
            m = render_frame(H, W, K, c2w, args.near, args.far, model_coarse, model_fine, N_samples=args.N_samples,
                             N_importance=args.N_importance, device=dev, keep_objects=kept, impl=impl, region=region,
                             appearance=appearance)
            m = {k: v.to(dev) for k, v in m.items()}
            out.append(m)
            if savedir is not None:
                rgba = np.concatenate([_to8b(m["rgb"].cpu().numpy()), _to8b(m["acc"].cpu().numpy())[..., None]], -1)
                write_png(os.path.join(savedir, "{:03d}.png".format(i)), rgba)
                from .mesh import argmax_rows
                label = argmax_rows(m["ins"].reshape(H * W, -1)).reshape(H, W)
                write_png(os.path.join(savedir, "instance_{:03d}.png".format(i)), colorize(label, lut).cpu().numpy())
    return out


# ----------------------------------------------------------------------------------------------------------------- meshes
def occupancy_objects(model, scene_transform, keep_words, grid_dim=256, extents=None, near=4.0, far=15.0, N_importance=128,
                      slab=0, device="cuda"):
    """The occupancy sweep of mesh.occupancy_grid with the selection applied per grid point -> (occ [dim]^3 float32, labels
    [dim]^3 int16): occ is 0 where the point's label is not kept, labels is every point's label."""
    from .mesh import EXTENTS, _sweep
    return _sweep(model, scene_transform, grid_dim, EXTENTS if extents is None else extents, near, far, N_importance, slab, device,
                  keep_words)


def meshes_from_labelled_grid(occ, labels, scene_transform, objects, level=0.45, extents=None, min_cluster=400):
    """The per-object stage: for each label k of `objects`, the field where(labels == k, occ, 0) -> marching cubes -> scene space
    -> vertex normals -> small-cluster removal.  Returns {k: {"vertices", "triangles", "normals" (the marching-cubes mesh),
    "clean_vertices", "clean_normals", "clean_triangles"}} of device tensors.  The field is 0 outside the object, so its mesh is
    closed wherever the object does not touch the grid boundary."""
    from .mesh import EXTENTS, clean_mesh, marching_cubes, to_scene, vertex_normals
    extents = EXTENTS if extents is None else extents
    dim = occ.shape[0]
    zero = torch.zeros((), device=occ.device, dtype=occ.dtype)
    out = {}
    for k in objects:
        field = torch.where(labels == int(k), occ, zero)
        v_idx, tris = marching_cubes(field, level)
        del field
        verts = to_scene(v_idx, scene_transform, dim, extents)
        if tris.shape[0] == 0:
            normals = torch.zeros_like(verts)
            out[int(k)] = {"vertices": verts, "triangles": tris, "normals": normals, "clean_vertices": verts,
                           "clean_normals": normals, "clean_triangles": tris}
            continue
        normals = vertex_normals(verts, tris)
        cv, cn, ct = clean_mesh(verts, normals, tris, min_cluster)
        out[int(k)] = {"vertices": verts, "triangles": tris, "normals": normals, "clean_vertices": cv, "clean_normals": cn,
                       "clean_triangles": ct}
    return out


def object_meshes(model_fine, model_coarse, scene_transform, objects=None, grid_dim=256, level=0.45, extents=None, near=4.0,
                  far=15.0, N_importance=128, min_cluster=400, components=None):
    """One mesh per object: one selected occupancy sweep of model_fine (keeping `objects`) with the label grid, then
    meshes_from_labelled_grid.  objects: labels in [0, ins_num]; default every label present in the grid except the last
    channel (ins_num, "no object").  model_coarse is accepted for symmetry with extract_mesh and not evaluated: the labels come
    from the fine network's per-point logits, not from rendered rays.  components="largest": each object's field is occ on its
    largest 26-connected component (object_components at `level`) and 0 elsewhere.  Returns {label: mesh dict} of device
    tensors."""
    from .mesh import check_transform
    if components not in (None, "largest"):
        raise ValueError("object_meshes: components must be None or 'largest', got %r" % (components,))
    T = check_transform(scene_transform)
    dev = next(model_fine.parameters()).device
    ins_num = int(model_fine.ins_linear.weight.shape[0]) - 1
    with torch.no_grad():
        if objects is None:
            words = object_mask(ins_num, remove=[ins_num])
        else:
            objects = _labels(objects, ins_num, "object_meshes")
            words = object_mask(ins_num, keep=objects)
        occ, labels = occupancy_objects(model_fine, T, words, grid_dim, extents, near, far, N_importance, device=dev)
        if objects is None:
            objects = [k for k in torch.unique(labels).cpu().tolist() if k != ins_num]
        if components == "largest":
            labels = largest_component_grid(occ, labels, level, objects)
        return meshes_from_labelled_grid(occ, labels, T, objects, level, extents, min_cluster)


# ----------------------------------------------------------------------------------------------------------------- edited meshes
# DESIGN.md, "Meshing an edited scene": the moves of manipulator_eval / manipulate_frame applied per grid point to the labelled
# keep-all sweep, so that an edited scene can be meshed.  The network runs only at the target points inside each move's box.
EMPTY_BOX = (1, 0, 1, 0, 1, 0)       # the inventory's box of a group without points: a move with it evaluates nothing


def _move_matrix(trans, i):
    m = np.asarray(trans, dtype=np.float64)
    if m.shape != (4, 4) or not np.isfinite(m).all():
        raise ValueError("edit: move %d: the transformation must be a finite 4x4 matrix, got shape %s" % (i, m.shape))
    if not np.array_equal(m[3], [0.0, 0.0, 0.0, 1.0]):
        raise ValueError("edit: move %d: the transformation's last row must be (0, 0, 0, 1)" % i)
    if np.linalg.det(m[:3, :3]) <= 0:
        raise ValueError("edit: move %d: the transformation has a non-positive determinant (a reflection or a degenerate "
                         "matrix)" % i)
    return m


def _check_moves(moves, ins_num):
    """moves [(label, 4x4)] -> (labels, matrices); ValueError for more than MAX_MOVES, a label outside [0, ins_num] or a bad
    matrix.  A matrix may be manipulation_transform(...)["transformations"][0]["transformation"] (a nested list)."""
    moves = list(moves)
    if len(moves) > _lib.MAX_MOVES:
        raise ValueError("edit: at most %d moves are supported, got %d" % (_lib.MAX_MOVES, len(moves)))
    labels, mats = [], []
    for i, mv in enumerate(moves):
        try:
            label, trans = mv
        except (TypeError, ValueError):
            raise ValueError("edit: move %d must be a pair (label, 4x4 transformation)" % i) from None
        labels.append(_labels([label], ins_num, "edit")[0])
        mats.append(_move_matrix(trans, i))
    return labels, mats


def _check_level(level):
    level = float(level)
    if not 0.0 < level < 1.0:
        raise ValueError("edit: level %r outside (0, 1)" % level)
    return level


def _check_boxes(boxes, m, dim):
    b = np.asarray(boxes, dtype=np.int64)
    if b.shape != (m, 6):
        raise ValueError("edit: boxes must be [%d, 6] inclusive index boxes, got shape %s" % (m, b.shape))
    for i in range(m):
        if tuple(b[i]) == EMPTY_BOX:
            continue
        if not all(0 <= b[i, 2 * a] <= b[i, 2 * a + 1] <= dim - 1 for a in range(3)):
            raise ValueError("edit: box %d %s is inverted or outside the grid [0, %d]" % (i, b[i].tolist(), dim - 1))
    return b


def _region_keeps(region, T, dim, extents, device, slab=1 << 20):
    """bool [dim]^3: the sweep grid points a piece keeps for a label it applies to -- inside its grid with the bit set, or
    outside it when it keeps outside samples -- by the render kernels' own test (region_contains)."""
    from .mesh import EXTENTS, grid_points
    ext = EXTENTS if extents is None else extents
    whole = None
    if region.outside == "keep":
        words = np.full((region.dim ** 3 + 31) // 32, -1, dtype=np.int32)
        tail = region.dim ** 3 % 32
        if tail:
            words[-1] = (1 << tail) - 1
        whole = Region(torch.as_tensor(words).to(region.bits.device), region.dim, region.voxel_map, region.applies, "keep")
    keep = torch.empty(dim ** 3, dtype=torch.bool, device=device)
    for b in range(0, dim ** 3, slab):
        pts = grid_points(T, dim, ext, b, min(slab, dim ** 3 - b), device)
        k = region_contains(region, pts)
        if whole is not None:
            k |= ~region_contains(whole, pts)
        keep[b:b + pts.shape[0]] = k
    return keep.reshape((dim,) * 3)


def solid_box(occ, labels, label, level=0.45, margin=2, keep=None):
    """The inclusive index box (i_lo, i_hi, j_lo, j_hi, k_lo, k_hi) of the solid points (occ > level) of `label` (and of `keep`,
    a bool grid, when given), grown by `margin` voxels on every side and clipped to the grid; EMPTY_BOX without points."""
    mask = (labels == int(label)) & (occ > level)
    if keep is not None:
        mask &= keep
    if not bool(mask.any()):
        return EMPTY_BOX
    dim = occ.shape[0]
    box = []
    for a in range(3):
        idx = torch.nonzero(mask.any(dim=tuple(c for c in range(3) if c != a))).flatten()
        box += [max(int(idx[0]) - int(margin), 0), min(int(idx[-1]) + int(margin), dim - 1)]
    return tuple(box)


def edit_occupancy(model_fine, scene_transform, occ, labels, moves, boxes, extents=None, level=0.45, near=4.0, far=15.0,
                   N_importance=128, pieces=None, rest="keep", slab=0):
    """dmnerf_mesh_occupancy_edit: the moves [(label, 4x4)] applied in order, in place, to occ / labels ([dim]^3 float32 /
    int16 on the device: the keep-all sweep of model_fine on this grid), the network evaluated only at the target points
    inside each move's box (boxes: [m, 6] inclusive index boxes, EMPTY_BOX for none).  pieces / rest: as manipulator.  Returns
    the number of target points evaluated."""
    from .manipulator import _piece_region, move_pieces, move_rests
    from .mesh import EXTENTS, check_transform
    T = check_transform(scene_transform)
    dim = _check_grid(occ, labels, "edit_occupancy")
    if labels is None or labels.dtype != torch.int16 or occ.dtype != torch.float32:
        raise ValueError("edit_occupancy: occ must be float32 and labels int16")
    ins_num = int(model_fine.ins_linear.weight.shape[0]) - 1
    mv, mats = _check_moves(moves, ins_num)
    level = _check_level(level)
    boxes = _check_boxes(boxes, len(mv), dim)
    drops = move_rests(rest, len(mv))
    regions = move_pieces(pieces, mv, ins_num, occ.device) or [None] * len(mv)
    if not mv:
        return 0
    descs = (_lib.EditMove * len(mv))()
    for i in range(len(mv)):
        d = descs[i]
        d.label, d.rest_drop = mv[i], int(drops[i])
        d.trans[:] = mats[i][:3].reshape(-1).tolist()
        d.box[:] = [int(v) for v in boxes[i]]
        d.piece = _piece_region(regions[i], mv[i], ins_num, occ.device)
    ctx = get_context(occ.device)
    slot = ctx.slot_for(model_fine)
    ctx.bind(slot, model_fine)
    ext = EXTENTS if extents is None else extents
    n = C.c_int64(0)
    with torch.no_grad():
        ctx.call("dmnerf_mesh_occupancy_edit", ctx.handle, slot, _lib.doubles(T, 16), _lib.doubles(ext, 3), dim,
                 (far - near) / N_importance, level, int(slab), descs, len(mv), _lib.ptr(occ), _lib.ptr(labels, torch.int16),
                 C.byref(n))
    return int(n.value)


def edit_boxes(occ, labels, moves, scene_transform, extents=None, level=0.45, margin=2, pieces=None):
    """The default boxes of edited_sweep from the unedited sweep: per move, solid_box of its label's solid points (those its
    piece keeps, with a piece) grown by margin -> int [m, 6]."""
    if int(margin) != margin or int(margin) < 0:
        raise ValueError("edit: margin must be an integer >= 0, got %r" % (margin,))
    mv = [int(m[0]) for m in moves]
    regions = list(pieces) if pieces is not None else [None] * len(mv)
    dim = occ.shape[0]
    out = []
    for k, r in zip(mv, regions):
        keep = None if r is None else _region_keeps(r, scene_transform, dim, extents, occ.device)
        out.append(solid_box(occ, labels, k, level, int(margin), keep))
        del keep
    return np.asarray(out, dtype=np.int64).reshape(len(mv), 6)


def edited_sweep(model_fine, scene_transform, moves, grid_dim=256, extents=None, level=0.45, near=4.0, far=15.0, N_importance=128,
                 margin=2, boxes=None, pieces=None, rest="keep"):
    """The labelled sweep of the edited scene -> (occ [dim]^3 float32, labels [dim]^3 int16) on the device: the keep-all sweep of
    model_fine (occupancy_objects), then the moves [(label, 4x4 in the network frame, as manipulator_eval's transformation)]
    applied in order (edit_occupancy).  A move shows at p what the network holds at trans p, as rigid_rays renders it: the
    object lands at inv(trans) x.  boxes: per move the index box of the target points evaluated; by default the box of the
    moved label's solid points in the unedited grid (of those its piece keeps, with a piece) grown by `margin` voxels.
    pieces / rest: as manipulator (a Region or None per move; "keep" / "drop", or one per move)."""
    from .manipulator import move_pieces, move_rests
    from .mesh import check_transform
    T = check_transform(scene_transform)
    dev = next(model_fine.parameters()).device
    ins_num = int(model_fine.ins_linear.weight.shape[0]) - 1
    mv, _ = _check_moves(moves, ins_num)
    level = _check_level(level)
    move_rests(rest, len(mv))
    move_pieces(pieces, mv, ins_num, dev)
    if int(margin) != margin or int(margin) < 0:
        raise ValueError("edit: margin must be an integer >= 0, got %r" % (margin,))
    if boxes is not None:
        boxes = _check_boxes(boxes, len(mv), int(grid_dim))
    with torch.no_grad():
        occ, labels = occupancy_objects(model_fine, T, object_mask(ins_num, remove=[]), grid_dim, extents, near, far, N_importance,
                                        device=dev)
        if boxes is None:
            boxes = edit_boxes(occ, labels, moves, T, extents, level, margin, pieces)
        edit_occupancy(model_fine, T, occ, labels, moves, boxes, extents, level, near, far, N_importance, pieces, rest)
    return occ, labels


def edited_mesh(model_fine, scene_transform, moves, grid_dim=256, extents=None, level=0.45, near=4.0, far=15.0, N_importance=128,
                margin=2, boxes=None, pieces=None, rest="keep", min_cluster=400, per_object=False):
    """The mesh of an edited scene: edited_sweep (same arguments) -> marching cubes -> scene space -> normals -> small-cluster
    removal.  Returns extract_mesh's keys as device tensors -- vertices, triangles, normals, clean_vertices, clean_normals,
    clean_triangles -- and labels (int64 per clean vertex: mesh.vertex_labels of its index-space vertex, the label of the
    inside end of its edge, from the edited grid; no label rays are rendered).  per_object: also objects, the
    meshes_from_labelled_grid of the edited grid for every label with solid points except ins_num."""
    from .mesh import EXTENTS, check_transform, clean_mesh, marching_cubes, to_scene, vertex_labels, vertex_normals
    T = check_transform(scene_transform)
    ext = EXTENTS if extents is None else extents
    ins_num = int(model_fine.ins_linear.weight.shape[0]) - 1
    with torch.no_grad():
        occ, labels = edited_sweep(model_fine, T, moves, grid_dim, ext, level, near, far, N_importance, margin, boxes, pieces, rest)
        v_idx, tris = marching_cubes(occ, level)
        verts = to_scene(v_idx, T, grid_dim, ext)
        normals = vertex_normals(verts, tris)
        cv, cn, ct = clean_mesh(verts, normals, tris, min_cluster)
        ci, _, _ = clean_mesh(v_idx, None, tris, min_cluster)         # the same topological cleanup, index space
        out = {"vertices": verts, "triangles": tris, "normals": normals, "clean_vertices": cv, "clean_normals": cn,
               "clean_triangles": ct, "labels": vertex_labels(ci, occ, labels, level).long()}
        if per_object:
            objects = [k for k in torch.unique(labels[occ > level]).cpu().tolist() if k != ins_num]
            out["objects"] = meshes_from_labelled_grid(occ, labels, T, objects, level, ext, min_cluster)
    return out


def largest_component_grid(occ, labels, level, objects):
    """int16 grid: label k at the points of the largest 26-connected component of each label k of `objects`, -1 elsewhere."""
    cc = object_components(occ, labels, level, 26)
    best = largest_components(cc["label"], cc["voxels"])
    lut = np.full(cc["label"].shape[0], -1, dtype=np.int16)
    for k in objects:
        if int(k) in best:
            lut[best[int(k)]] = int(k)
    return component_groups(cc["grid"], lut, -1)


# ----------------------------------------------------------------------------------------------------------------- inventory
# DESIGN.md, "Object inventory": which objects the model found and where they are, from the solid points (occ > level) of a
# labelled sweep.  Every statistic is taken over an object's points: its solid points inside its trimmed index box.
MESH_TO_NETWORK = np.array([[1.0, 0.0, 0.0], [0.0, 0.0, -1.0], [0.0, 1.0, 0.0]])    # (x, y, z) -> (x, -z, y), grid_points_kernel
N_MOMENTS = 10                       # count, Si, Sj, Sk, Sii, Sjj, Skk, Sij, Sik, Sjk


def grid_affine(scene_transform, dim, extents=None):
    """The exact map from grid index (i, j, k) to the network frame, p = A @ idx + b, in fp64: linspace(-1, 1, dim) scaled by
    extents / 2, then [R | t], then the axis swap of the sweep.  The sweep's fp32 grid points differ from it by fp32 rounding."""
    from .mesh import EXTENTS, check_transform
    T = check_transform(scene_transform)
    ext = np.asarray(EXTENTS if extents is None else extents, dtype=np.float64).reshape(3)
    R, t = T[:3, :3], T[:3, 3]
    A = MESH_TO_NETWORK @ (R * (ext / (dim - 1))[None, :])
    b = MESH_TO_NETWORK @ (t - R @ (ext / 2.0))
    return A, b


def _check_grid(occ, labels, who):
    _lib.need_cuda(who, occ, labels)
    if occ.dim() != 3 or not (occ.shape[0] == occ.shape[1] == occ.shape[2]):
        raise ValueError("%s: occ must be a cubic grid [dim, dim, dim], got %s" % (who, tuple(occ.shape)))
    if labels is not None and (labels.shape != occ.shape or labels.device != occ.device):
        raise ValueError("%s: labels must have occ's shape and device" % who)
    return occ.shape[0]


def object_voxels(occ, labels, level, n_labels, boxes=None):
    """dmnerf_object_voxels: per group 0 .. n_labels - 1 (labels None: one group) the integer moments [n_labels, 10] int64
    (count, Si, Sj, Sk, Sii, Sjj, Skk, Sij, Sik, Sjk of the index coordinates) and the per-axis index histograms
    [n_labels, 3, dim] uint32 of its solid points, inside its box when boxes ([n_labels, 6] inclusive index boxes) is given."""
    dim = _check_grid(occ, labels, "object_voxels")
    ctx = get_context(occ.device)
    mom = np.zeros((n_labels, N_MOMENTS), dtype=np.int64)
    hist = np.zeros((n_labels, 3, dim), dtype=np.uint32)
    ctx.call("dmnerf_object_voxels", ctx.handle, _lib.ptr(occ), _lib.ptr(labels, torch.int16), dim, float(level), int(n_labels),
             _int32s(boxes, n_labels * 6), mom.ctypes.data_as(C.POINTER(C.c_int64)), hist.ctypes.data_as(C.POINTER(C.c_uint32)))
    return mom, hist


def object_spans(occ, labels, level, n_labels, boxes, axes):
    """dmnerf_object_spans: per group and axis r the min and max over its points (solid, inside its box) of
    ((u0 i + u1 j) + u2 k) + o with axes[g, r] = (u0, u1, u2, o), fp64 -> [n_labels, 3, 2]; (+inf, -inf) without points."""
    _check_grid(occ, labels, "object_spans")
    ctx = get_context(occ.device)
    out = np.zeros((n_labels, 3, 2), dtype=np.float64)
    ctx.call("dmnerf_object_spans", ctx.handle, _lib.ptr(occ), _lib.ptr(labels, torch.int16), occ.shape[0], float(level),
             int(n_labels), _int32s(boxes, n_labels * 6), _lib.doubles(axes, n_labels * 12), out.ctypes.data_as(C.POINTER(C.c_double)))
    return out


def _int32s(a, n):
    return None if a is None else (C.c_int32 * n)(*np.asarray(a, dtype=np.int64).reshape(-1).tolist())


def trimmed_boxes(hist, trim):
    """Per group and grid axis, the index range [lo, hi] left after cutting floor(trim * N) of the N solid points from each end
    of that axis's histogram -> int32 [n_groups, 6] (i_lo, i_hi, j_lo, j_hi, k_lo, k_hi); a group without points gets (1, 0)."""
    hist = np.asarray(hist, dtype=np.int64)
    out = np.zeros((hist.shape[0], 6), dtype=np.int32)
    for g in range(hist.shape[0]):
        n = int(hist[g, 0].sum())
        if n == 0:
            out[g] = (1, 0) * 3
            continue
        cut = int(np.floor(trim * n))
        for a in range(3):
            c = np.cumsum(hist[g, a])
            out[g, 2 * a] = int(np.argmax(c > cut))                                  # first index with more than cut below it
            out[g, 2 * a + 1] = int(np.nonzero(c < n - cut)[0].size)                  # first index with more than cut above it
    return out


def _check_trim(trim):
    trim = float(trim)
    if not 0.0 <= trim < 0.5:
        raise ValueError("trim %r outside [0, 0.5)" % trim)
    return trim


def describe_groups(moments, boxes, A, b, voxel_volume, groups):
    """The host stage of the inventory: for each group of `groups` with points, its entry from the integer moments of its
    points and its box -> (entries, spans axes [n, 3, 4]).  The OBB half-sizes come from finish_obbs."""
    entries = []
    axes_in = np.zeros((moments.shape[0], 3, 4))
    for g in groups:
        n = int(moments[g, 0])
        if n == 0:
            continue
        s = [int(v) for v in moments[g]]
        S1 = s[1:4]
        S2 = [[s[4], s[7], s[8]], [s[7], s[5], s[9]], [s[8], s[9], s[6]]]
        mean = np.array([S1[a] / n for a in range(3)])
        cov_idx = np.array([[(n * S2[a][c] - S1[a] * S1[c]) / (n * n) for c in range(3)] for a in range(3)])
        centre = A @ mean + b
        cov = A @ cov_idx @ A.T
        lo, hi = boxes[g, 0::2].astype(np.float64), boxes[g, 1::2].astype(np.float64)
        corners = np.array([[(hi if (c >> a) & 1 else lo)[a] for a in range(3)] for c in range(8)]) @ A.T + b
        w, V = np.linalg.eigh(cov)
        axes = V[:, ::-1].T.copy()                                  # rows, descending eigenvalue
        for r in range(2):
            if axes[r, np.argmax(np.abs(axes[r]))] < 0:
                axes[r] = -axes[r]
        axes[2] = np.cross(axes[0], axes[1])
        axes_in[g, :, :3] = axes @ A
        axes_in[g, :, 3] = axes @ (b - centre)
        entries.append({"label": int(g), "voxels": n, "volume": n * voxel_volume, "centre": centre, "covariance": cov,
                        "aabb": (corners.min(0), corners.max(0)), "box": boxes[g].copy(),
                        "obb": {"axes": axes, "eigenvalues": w[::-1].copy()}})
    return entries, axes_in


def finish_obbs(entries, spans):
    """OBB centre and half-sizes of every entry from its spans [n, 3, 2] (min, max of the projections on its axes)."""
    for e in entries:
        lo, hi = spans[e["label"], :, 0], spans[e["label"], :, 1]
        e["obb"]["centre"] = e["centre"] + e["obb"]["axes"].T @ ((lo + hi) / 2.0)
        e["obb"]["half_sizes"] = (hi - lo) / 2.0
    return entries


def _inventory_of_groups(occ, labels, n_labels, T, ext, dim, level, trim, groups):
    """The device passes and host stage of inventory_from_grid over the groups of one group grid (labels, n_labels)."""
    mom, hist = object_voxels(occ, labels, level, n_labels)
    boxes = trimmed_boxes(hist, trim)
    if trim > 0:
        mom, _ = object_voxels(occ, labels, level, n_labels, boxes)
    A, b = grid_affine(T, dim, ext)
    unit = abs(np.linalg.det(T[:3, :3])) * float(np.prod(ext / (dim - 1)))
    entries, axes_in = describe_groups(mom, boxes, A, b, unit, groups)
    if not entries:
        return []
    spans = object_spans(occ, labels, level, n_labels, boxes, axes_in)
    return finish_obbs(entries, spans)


def inventory_from_grid(occ, labels, scene_transform, extents=None, level=0.45, trim=0.0, objects=None, components=None,
                        connectivity=26, min_voxels=1):
    """The grid-only stage of object_inventory: occ [dim]^3 float32 and labels [dim]^3 int16 (or None: one group, the scene)
    on the device.  Returns one entry per group (of `objects`, default all) that has points, ascending label:
      label, voxels, volume (voxels |det R| prod(extents / (dim - 1))), centre and covariance (network frame),
      aabb (min, max of the trimmed box's corners, network frame), box (the trimmed index box),
      obb {centre, axes (rows: eigenvectors of the covariance, descending eigenvalue, right-handed), eigenvalues, half_sizes}.
    components (DESIGN.md, "Connected components"; `connectivity` 6 or 26):
      None:      a label is one object;
      "largest": each label's statistics over its largest component only (a tie in voxels goes to the smaller root); the
                 entry gains components (how many the label has) and discarded_voxels (its solid points outside that one);
      "split":   one entry per component with at least min_voxels voxels, ordered by (label, root), with component (its id).
    trim applies after the selection, over the selected points.  An edited grid (edited_sweep) is a labelled grid like any
    other: its inventory reports the objects where the moves put them."""
    from .mesh import EXTENTS, check_transform
    trim = _check_trim(trim)
    if components not in (None, "largest", "split"):
        raise ValueError("inventory_from_grid: components must be None, 'largest' or 'split', got %r" % (components,))
    if int(min_voxels) < 1 or (int(min_voxels) != 1 and components != "split"):
        raise ValueError("inventory_from_grid: min_voxels %r needs components='split' and must be >= 1" % (min_voxels,))
    T = check_transform(scene_transform)
    ext = np.asarray(EXTENTS if extents is None else extents, dtype=np.float64).reshape(3)
    dim = _check_grid(occ, labels, "inventory_from_grid")
    n_labels = MAX_LABELS if labels is not None else 1
    groups = range(n_labels) if objects is None else sorted({int(k) for k in objects})
    if any(not 0 <= g < n_labels for g in groups):
        raise ValueError("inventory_from_grid: objects must be labels in [0, %d]" % (n_labels - 1))
    with torch.no_grad():
        if components is None:
            return _inventory_of_groups(occ, labels, n_labels, T, ext, dim, level, trim, groups)
        cc = object_components(occ, labels, level, connectivity)
        sel = select_components(cc["label"], cc["voxels"], components, groups, int(min_voxels))
        entries = []
        for lut, ids in group_luts(sel, cc["label"].shape[0]):
            grid = component_groups(cc["grid"], lut, DISCARD_GROUP)
            part = _inventory_of_groups(occ, grid, MAX_LABELS, T, ext, dim, level, trim, range(len(ids)))
            del grid
            for e in part:
                c = int(ids[e["label"]])
                e["label"] = int(cc["label"][c])
                if components == "largest":
                    same = cc["label"] == e["label"]
                    e["components"] = int(np.count_nonzero(same))
                    e["discarded_voxels"] = int(cc["voxels"][same].sum() - cc["voxels"][c])
                else:
                    e["component"] = c
            entries += part
    return entries


def object_inventory(model_fine, scene_transform, extents=None, grid_dim=256, level=0.45, trim=0.0, objects=None, near=4.0,
                     far=15.0, N_importance=128, components=None, connectivity=26, min_voxels=1):
    """Which objects the model found and where: one selected occupancy sweep of model_fine (keeping `objects`, default every
    label except ins_num, as object_meshes) with its label grid, then inventory_from_grid (components, connectivity and
    min_voxels as there)."""
    from .mesh import check_transform
    T = check_transform(scene_transform)
    dev = next(model_fine.parameters()).device
    ins_num = int(model_fine.ins_linear.weight.shape[0]) - 1
    objects = list(range(ins_num)) if objects is None else _labels(objects, ins_num, "object_inventory")
    with torch.no_grad():
        occ, labels = occupancy_objects(model_fine, T, object_mask(ins_num, keep=objects), grid_dim, extents, near, far,
                                        N_importance, device=dev)
        return inventory_from_grid(occ, labels, T, extents, level, trim, objects, components, connectivity, min_voxels)


# ----------------------------------------------------------------------------------------------------------------- components
# DESIGN.md, "Connected components": the solid points of a labelled grid split into components, numbered by their smallest
# C-order index; the inventory runs on a group grid that maps the chosen components to groups 0 .. 126 and the rest to 127.
GROUP_BATCH = MAX_LABELS - 1         # components per inventory batch
DISCARD_GROUP = MAX_LABELS - 1       # the group of every point outside the batch


def object_components(occ, labels=None, level=0.45, connectivity=26):
    """dmnerf_object_components + dmnerf_component_table: the connected components of the solid points (occ > level) of
    occ [dim]^3 float32, adjacency within one label of labels [dim]^3 int16 (None: one label) -> {"grid": int32 [dim]^3 on the
    device (component id, -1 where not solid), "label": int16 [n], "voxels": int64 [n], "root": int64 [n] (the component's
    smallest C-order linear index)}; ids ascend with the root.  An edited grid (edited_sweep) is accepted unchanged."""
    dim = _check_grid(occ, labels, "object_components")
    ctx = get_context(occ.device)
    grid = torch.empty(occ.shape, dtype=torch.int32, device=occ.device)
    n = C.c_int64(0)
    ctx.call("dmnerf_object_components", ctx.handle, _lib.ptr(occ), _lib.ptr(labels, torch.int16), dim, float(level),
             MAX_LABELS if labels is not None else 1, int(connectivity), _lib.ptr(grid, torch.int32), C.byref(n))
    n = int(n.value)
    label = torch.empty(n, dtype=torch.int16, device=occ.device)
    voxels = torch.empty(n, dtype=torch.int64, device=occ.device)
    root = torch.empty(n, dtype=torch.int64, device=occ.device)
    ctx.call("dmnerf_component_table", ctx.handle, _lib.ptr(grid, torch.int32), _lib.ptr(labels, torch.int16), dim, n,
             _lib.ptr(label, torch.int16), _lib.ptr(voxels, torch.int64), _lib.ptr(root, torch.int64))
    return {"grid": grid, "label": label.cpu().numpy(), "voxels": voxels.cpu().numpy(), "root": root.cpu().numpy()}


def component_groups(grid, lut, discard):
    """dmnerf_component_groups: the int16 group grid lut[id] of a component id grid, `discard` where it is -1 (not solid)."""
    _lib.need_cuda("component_groups", grid)
    lut = torch.as_tensor(np.asarray(lut, dtype=np.int16)).to(grid.device)
    out = torch.empty(grid.shape, dtype=torch.int16, device=grid.device)
    ctx = get_context(grid.device)
    ctx.call("dmnerf_component_groups", ctx.handle, _lib.ptr(grid, torch.int32), grid.shape[0], lut.shape[0],
             _lib.ptr(lut, torch.int16), int(discard), _lib.ptr(out, torch.int16))
    return out


def largest_components(label, voxels):
    """{label: id of its largest component}; on a tie in voxels the smaller id (the smaller root) wins."""
    label, voxels = np.asarray(label, dtype=np.int64), np.asarray(voxels, dtype=np.int64)
    order = np.lexsort((np.arange(label.shape[0]), -voxels, label))       # by label, then most voxels, then smallest id
    first = np.ones(order.shape[0], dtype=bool)
    first[1:] = label[order][1:] != label[order][:-1]
    return {int(label[c]): int(c) for c in order[first]}


def select_components(label, voxels, components, groups, min_voxels=1):
    """The component ids an inventory reports, in entry order: "largest": each label of `groups`' largest component, ascending
    label; "split": every component of a label of `groups` with at least min_voxels voxels, by (label, root)."""
    groups = set(int(g) for g in groups)
    if components == "largest":
        best = largest_components(label, voxels)
        return [best[k] for k in sorted(best) if k in groups]
    label, voxels = np.asarray(label, dtype=np.int64), np.asarray(voxels, dtype=np.int64)
    ids = np.nonzero(np.isin(label, sorted(groups)) & (voxels >= min_voxels))[0]
    return [int(c) for c in ids[np.lexsort((ids, label[ids]))]]


def group_luts(ids, n_components):
    """Batches of GROUP_BATCH of the component ids `ids` -> [(lut int16 [n_components], batch ids)]: lut[batch[g]] = g, every
    other component DISCARD_GROUP."""
    out = []
    for s in range(0, len(ids), GROUP_BATCH):
        batch = list(ids[s:s + GROUP_BATCH])
        lut = np.full(n_components, DISCARD_GROUP, dtype=np.int16)
        lut[batch] = np.arange(len(batch), dtype=np.int16)
        out.append((lut, batch))
    return out


# ----------------------------------------------------------------------------------------------------------------- regions
# DESIGN.md, "Region selection": one bit per point of the sweep grid, read per sample by the render kernels.  A sample whose label
# is in the region's `applies` labels gets alpha = 0 when its nearest grid point's bit is 0, or when it lies outside the grid and
# `outside` is "drop".
REGION_MAX_DIM = 1290                # dim^3 < 2^31, as object_components


def voxel_map(scene_transform, dim, extents=None):
    """The fp32 map [M | c] (3x4) from the network frame to grid indices of the sweep grid: grid_affine (A, b) in fp64, M =
    inv(A), c = -inv(A) b, each of the 12 numbers rounded once to fp32."""
    A, b = grid_affine(scene_transform, dim, extents)
    M = np.linalg.inv(A)
    return np.concatenate([M, (-M @ b)[:, None]], 1).astype(np.float32)


class Region:
    """A region of the sweep grid: bits (int32 CUDA tensor, ceil(dim^3 / 32) words; point v = (i dim + j) dim + k is bit v & 31
    of word v >> 5), dim, voxel_map (float32 [3, 4], voxel_map()), applies (the 4 label words it applies to, or None: every
    label of the networks it renders with) and outside ("keep" or "drop": samples outside the grid)."""

    def __init__(self, bits, dim, voxel_map, applies=None, outside="keep"):
        dim = int(dim)
        if not 2 <= dim <= REGION_MAX_DIM:
            raise ValueError("Region: dim %d outside [2, %d]" % (dim, REGION_MAX_DIM))
        words = (dim ** 3 + 31) // 32
        if not torch.is_tensor(bits) or bits.dtype != torch.int32 or not bits.is_cuda or bits.dim() != 1 or \
                bits.shape[0] != words or not bits.is_contiguous():
            raise ValueError("Region: bits must be a contiguous int32 CUDA tensor of %d words for dim %d" % (words, dim))
        vm = np.asarray(voxel_map, dtype=np.float32).reshape(3, 4)
        if not np.isfinite(vm).all():
            raise ValueError("Region: the voxel map is not finite")
        if outside not in ("keep", "drop"):
            raise ValueError("Region: outside must be 'keep' or 'drop', got %r" % (outside,))
        if applies is not None:
            applies = [int(w) & 0xFFFFFFFF for w in applies]
            if len(applies) != 4:
                raise ValueError("Region: applies takes 4 label words")
        self.bits, self.dim, self.voxel_map, self.applies, self.outside = bits, dim, vm, applies, outside

    def applies_words(self, ins_num):
        """The 4 label words for networks with ins_num: applies, or every label 0 .. ins_num."""
        return object_mask(ins_num, remove=[]) if self.applies is None else list(self.applies)

    def abi(self, ins_num):
        """The C ABI's dmnerf_region (_lib.RegionDesc) of this region for networks with ins_num.  It points at self.bits: keep
        this Region alive until the call that reads it returns."""
        d = _lib.RegionDesc(bits=_lib.ptr(self.bits, torch.int32).value, dim=self.dim, outside_keep=int(self.outside == "keep"))
        d.voxel_map[:] = [float(v) for v in np.asarray(self.voxel_map, dtype=np.float32).reshape(-1)]
        d.applies[:] = self.applies_words(ins_num)
        return d


def label_words(labels):
    """The 4 label words of an iterable of labels in [0, 127] (a region's applies)."""
    words = [0, 0, 0, 0]
    for k in labels:
        k = int(k)
        if not 0 <= k < MAX_LABELS:
            raise ValueError("label %d outside [0, %d]" % (k, MAX_LABELS - 1))
        words[k >> 5] |= 1 << (k & 31)
    return words


def _check_build(dilate, connectivity, outside):
    if int(dilate) != dilate or int(dilate) < 0:
        raise ValueError("region: dilate must be an integer >= 0, got %r" % (dilate,))
    if connectivity not in (6, 26):
        raise ValueError("region: connectivity %r is not 6 or 26" % (connectivity,))
    if outside not in ("keep", "drop"):
        raise ValueError("region: outside must be 'keep' or 'drop', got %r" % (outside,))


def _region_bits(ids, table, n_ids, dim, dilate, connectivity, invert):
    """dmnerf_region_pack of an int32 id grid with a table over ids, then dmnerf_region_dilate -> int32 words."""
    dilate, connectivity = int(dilate), int(connectivity)
    words = (dim ** 3 + 31) // 32
    packed = torch.empty(words, dtype=torch.int32, device=ids.device)
    ctx = get_context(ids.device)
    tab = torch.as_tensor(np.asarray(table, dtype=np.uint32).view(np.int32)).to(ids.device)
    ctx.call("dmnerf_region_pack", _lib.ptr(ids, torch.int32), dim, _lib.ptr(tab, torch.int32), int(n_ids),
             _lib.ptr(packed, torch.int32))
    if dilate == 0 and not invert:
        return packed
    out = torch.empty_like(packed)
    ctx.call("dmnerf_region_dilate", ctx.handle, _lib.ptr(packed, torch.int32), dim, dilate, connectivity, int(bool(invert)),
             _lib.ptr(out, torch.int32))
    return out


def _check_cube(grid, who):
    _lib.need_cuda(who, grid)
    if grid.dim() != 3 or not (grid.shape[0] == grid.shape[1] == grid.shape[2]):
        raise ValueError("%s: expected a cubic grid [dim, dim, dim], got %s" % (who, tuple(grid.shape)))
    dim = int(grid.shape[0])
    if not 2 <= dim <= REGION_MAX_DIM:
        raise ValueError("%s: dim %d outside [2, %d]" % (who, dim, REGION_MAX_DIM))
    return dim


def region_from_mask(mask, scene_transform, extents=None, applies=None, outside="keep", dilate=0, connectivity=26):
    """A Region from a boolean grid mask [dim]^3 (CUDA) over the sweep grid of (scene_transform, extents): the points where mask
    is True, grown by `dilate` dilation steps.  applies: labels it applies to (default every label); outside as in Region.  An
    index box [i0:i1, j0:j1, k0:k1] goes through here as a mask."""
    _check_build(dilate, connectivity, outside)
    dim = _check_cube(mask, "region_from_mask")
    ids = torch.where(mask.bool(), 0, -1).to(torch.int32).contiguous()
    bits = _region_bits(ids, [1], 1, dim, dilate, connectivity, False)
    return Region(bits, dim, voxel_map(scene_transform, dim, extents), None if applies is None else label_words(applies), outside)


def component_region(cc, ids, scene_transform, extents=None, dilate=1, connectivity=26, invert=False, outside="keep"):
    """A Region from components of object_components' result `cc`: the points of the components `ids`, grown by `dilate`
    dilation steps (`connectivity` 6 or 26), complemented when invert.  It applies to the labels of `ids` only.
      one piece alone:  component_region(cc, [j], T)                 -- drops every other piece of j's label
      one piece out:    component_region(cc, [j], T, invert=True)    -- drops piece j, keeps the rest of its label
      floater cleanup:  best = largest_components(cc["label"], cc["voxels"]);
                        component_region(cc, [best[k] for k in best if k != ins_num], T)
                        -- every object label keeps its largest piece (dilated by a voxel), its floaters go; labels as
                        object_inventory: every label but ins_num, from a sweep of object_inventory's selection."""
    _check_build(dilate, connectivity, outside)
    grid = cc["grid"]
    dim = _check_cube(grid, "component_region")
    n = int(np.asarray(cc["label"]).shape[0])
    ids = [int(c) for c in ids]
    if any(not 0 <= c < n for c in ids):
        raise ValueError("component_region: component ids must be in [0, %d)" % n)
    table = np.zeros(max(1, (n + 31) // 32), dtype=np.uint32)
    for c in ids:
        table[c >> 5] |= np.uint32(1 << (c & 31))
    bits = _region_bits(grid, table, n, dim, dilate, connectivity, invert)
    applies = label_words(sorted({int(cc["label"][c]) for c in ids}))
    return Region(bits, dim, voxel_map(scene_transform, dim, extents), applies, outside)


def region_contains(region, pts):
    """dmnerf_region_contains: bool [n] -- the point pts [n, 3] (network frame, CUDA) is inside the grid and its bit is set, by the
    render kernels' own test."""
    _lib.need_cuda("region_contains", pts)
    pts = pts.reshape(-1, 3).contiguous().float()
    out = torch.empty(pts.shape[0], dtype=torch.uint8, device=pts.device)
    desc = region.abi(MAX_LABELS - 1)                   # applies is not read here
    get_context(pts.device).call("dmnerf_region_contains", C.byref(desc), _lib.ptr(pts), pts.shape[0], _lib.ptr(out, torch.uint8))
    return out.bool()


# ----------------------------------------------------------------------------------------------------------------- appearance
# DESIGN.md, "Object appearance": per label a colour map and a density scale, applied per sample by the render kernels to every
# sample the selection and the region keep.
APPEARANCE_ROW = 16                  # floats per label: [M | b] row-major 3x4, the density scale, 3 of padding
LUMA = (0.299, 0.587, 0.114)


def tint(rgb):
    """The colour map (3x4, float64) that keeps a sample's shading and replaces its hue with rgb: c'_a = rgb_a (0.299 c0 +
    0.587 c1 + 0.114 c2), no offset.  tint((1, 1, 1)) is greyscale."""
    rgb = np.asarray(rgb, dtype=np.float64).reshape(-1)
    if rgb.shape != (3,) or not np.isfinite(rgb).all():
        raise ValueError("tint: rgb must be 3 finite numbers, got %r" % (rgb.tolist(),))
    return np.concatenate([np.outer(rgb, LUMA), np.zeros((3, 1))], 1)


class Appearance:
    """An object appearance for networks with ins_num: per label, the colour map [M | b] applied to a sample's sigmoid colour c
    (c' = clamp(M c + b, 0, 1)) and the scale s >= 0 of its density (alpha = 1 - exp(-s relu(sigma) dist)).
    colour: {label: 3x4 matrix [M | b], or 3x3 M (b = 0)}; density: {label: s}.  A label without an entry keeps its look
    (M = I, b = 0, s = 1).  `table` is the float32 [ins_num + 1, 16] table of dmnerf_edit.appearance."""

    def __init__(self, ins_num, colour=None, density=None):
        ins_num = int(ins_num)
        if not 1 <= ins_num <= MAX_LABELS - 1:
            raise ValueError("Appearance: ins_num %d outside [1, %d]" % (ins_num, MAX_LABELS - 1))
        table = np.zeros((ins_num + 1, APPEARANCE_ROW), dtype=np.float32)
        table[:, :12] = np.eye(3, 4, dtype=np.float32).reshape(12)
        table[:, 12] = 1.0
        for label, m in dict(colour or {}).items():
            k = _labels([label], ins_num, "Appearance")[0]
            m = np.asarray(m, dtype=np.float64)
            if m.shape == (3, 3):
                m = np.concatenate([m, np.zeros((3, 1))], 1)
            if m.shape != (3, 4):
                raise ValueError("Appearance: the colour map of label %d must be 3x4 or 3x3, got shape %s" % (k, m.shape))
            with np.errstate(over="ignore", invalid="ignore"):
                m = m.astype(np.float32)
            if not np.isfinite(m).all():
                raise ValueError("Appearance: the colour map of label %d is not finite in float32" % k)
            table[k, :12] = m.reshape(12)
        for label, s in dict(density or {}).items():
            k = _labels([label], ins_num, "Appearance")[0]
            with np.errstate(over="ignore", invalid="ignore"):
                s = np.float32(s)
            if not (np.isfinite(s) and s >= 0):
                raise ValueError("Appearance: the density scale of label %d must be finite and >= 0, got %r" % (k, float(s)))
            table[k, 12] = s
        self.ins_num, self.table = ins_num, table


def camera_region(poses, hwk, far):
    """Network-frame AABB (lo, hi) of the camera centres and of every camera's four corner rays at depth far: o + far * d with
    d = R ((u - cx) / fx, (v - cy) / fy, K[2, 2]), the direction get_rays_k gives pixel (u, v)."""
    H, W, K = hwk
    K = np.asarray(K, dtype=np.float64).reshape(3, 3)
    pts = []
    for c2w in poses:
        c2w = np.asarray(c2w.cpu() if torch.is_tensor(c2w) else c2w, dtype=np.float64)
        R, o = c2w[:3, :3], c2w[:3, 3]
        pts.append(o)
        for u in (0.0, float(W) - 1):
            for v in (0.0, float(H) - 1):
                d = R @ np.array([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], K[2, 2]])
                pts.append(o + far * d)
    pts = np.array(pts)
    return pts.min(0), pts.max(0)


def region_transform(lo, hi):
    """A network-frame AABB as (scene_transform, extents): box axes = the mesh-frame axes (det +1), network -> mesh is
    (x, y, z) -> (x, z, -y)."""
    lo, hi = np.asarray(lo, dtype=np.float64), np.asarray(hi, dtype=np.float64)
    m_lo = np.array([lo[0], lo[2], -hi[1]])
    m_hi = np.array([hi[0], hi[2], -lo[1]])
    T = np.eye(4)
    T[:3, 3] = (m_lo + m_hi) / 2.0
    return T, m_hi - m_lo


def box_transform(scene_transform, extents, dim, box):
    """The index box [lo, hi] (int [6]) of a grid with an axis-aligned transform (R = I) as (scene_transform, extents)."""
    T = np.asarray(scene_transform, dtype=np.float64)
    ext = np.asarray(extents, dtype=np.float64)
    step = ext / (dim - 1)
    lo, hi = np.asarray(box[0::2], dtype=np.float64), np.asarray(box[1::2], dtype=np.float64)
    out = np.eye(4)
    out[:3, 3] = T[:3, 3] - ext / 2.0 + step * (lo + hi) / 2.0
    return out, step * (hi - lo)


def scene_box(model_fine, poses, hwk, near, far, grid_dim=128, trim=1e-3, margin=2, level=0.45, N_importance=128):
    """The scene's box without a ground-truth mesh -> (scene_transform, extents) for extract_mesh / object_inventory:
    1. the camera region (camera_region), 2. one unselected coarse sweep over it, 3. the trimmed box of its solid points,
    padded by `margin` coarse voxels and kept inside the region.  A surface thinner than the coarse spacing can be missed:
    raise grid_dim (and margin) for thin scenes."""
    from .mesh import occupancy_grid
    trim = _check_trim(trim)
    if int(margin) < 0 or int(grid_dim) < 2:
        raise ValueError("scene_box: margin must be >= 0 and grid_dim >= 2")
    dev = next(model_fine.parameters()).device
    T0, ext0 = region_transform(*camera_region(poses, hwk, far))
    with torch.no_grad():
        occ = occupancy_grid(model_fine, T0, grid_dim, ext0, near, far, N_importance, device=dev)
        mom, hist = object_voxels(occ, None, level, 1)
    if mom[0, 0] == 0:
        raise ValueError("scene_box: no grid point of the camera region has occupancy above %g" % level)
    box = trimmed_boxes(hist, trim)[0].astype(np.int64)
    box[0::2] = np.maximum(box[0::2] - int(margin), 0)
    box[1::2] = np.minimum(box[1::2] + int(margin), grid_dim - 1)
    for a in range(3):                                  # at least one coarse spacing along every axis
        if box[2 * a] == box[2 * a + 1]:
            if box[2 * a + 1] < grid_dim - 1:
                box[2 * a + 1] += 1
            else:
                box[2 * a] -= 1
    return box_transform(T0, ext0, grid_dim, box)


def manipulation_transform(centre, mode, distance=-0.25, yaw=90.0, scale=1.2):
    """The transformation dict of the original's generate_poses_eval (tools/pose_generator.py) about `centre` (network frame):
    {'transformations': [{'transformation': 4x4 list, 'mode': mode}]}; mode translation (along y by distance), rotation (yaw
    degrees about z), scale, or multi (scale @ rotation @ translation).  As there, the centre is held in float32 and the
    products are taken in float64, so manipulator_eval receives the same matrix the original would build."""
    if mode not in ("translation", "rotation", "scale", "multi"):
        raise ValueError("manipulation_transform: unknown mode %r" % (mode,))
    c = np.asarray(centre, dtype=np.float64).reshape(3)
    to_origin = np.eye(4, dtype=np.float32)
    to_origin[:3, 3] = -c
    back = np.eye(4, dtype=np.float32)
    back[:3, 3] = -to_origin[:3, 3]
    move = np.eye(4)
    move[1, 3] = distance
    a = yaw * np.pi / 180
    turn = np.array([[np.cos(a), -np.sin(a), 0, 0], [np.sin(a), np.cos(a), 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    grow = np.diag([scale, scale, scale, 1.0])
    op = {"translation": move, "rotation": turn, "scale": grow, "multi": grow @ turn @ move}[mode]
    return {"transformations": [{"transformation": (back @ op @ to_origin).tolist(), "mode": mode}]}
