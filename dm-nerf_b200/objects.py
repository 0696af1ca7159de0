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
    move_overlap(occ, labels, scene_transform, moves, ...) / slide_until_contact(...) / object_contacts(...) / supports(...)
                                                        -> collision checks of moves, and which objects touch, from a sweep
    placement_map(occ, labels, scene_transform, label, down, ...) / placement(map, u, v) / place_object(..., near, ...)
                                                        -> where a lowered object comes to rest, on what, and whether it stands
    edited_grid(occ, labels, scene_transform, moves, ...) / arrange_objects(occ, labels, scene_transform, items, down, ...)
                                                        -> moves applied to the sweep alone, and several objects placed in turn
    render_moves(occ, labels, scene_transform, moves, ...)
                                                        -> moves for render_rays(moves=) / render_frame(moves=): the edited
                                                           sweep's rule applied per render sample
    carried_labels(occ, labels, scene_transform, label, down, ...)
                                                        -> what rests on an object, transitively: the group= that moves
                                                           it together with what it carries
    cast_grid(occ, labels, scene_transform, rays_o, rays_d, near, far, ...) / grid_view(occ, labels, scene_transform, H, W, K,
              c2w, near, far, ...)                     -> the first solid voxel along each ray (depth, label, voxel, normal,
                                                           piece), and depth, label, normal and colour maps of the grid
                                                           from one or several cameras, with no network; with moves= and
                                                           source=, an edited grid's hits traced to the moves that placed
                                                           them and coloured from the network at their source

Every network sample is labelled argmax(sigmoid(instance logits)) over all ins_num + 1 channels, first maximum winning (the
exchanger's rule); a sample whose label is not kept has alpha = 0 in the composite of both passes, so the coarse weights of the
selected scene drive the importance sampling.  The instance map keeps the network's channels: selection does not re-label it."""
import ctypes as C
import os
from fractions import Fraction

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


def _check_moves(moves, ins_num, limit=_lib.MAX_MOVES):
    """moves [(label, 4x4)] -> (labels, matrices); ValueError for more than `limit`, a label outside [0, ins_num] or a bad
    matrix.  A matrix may be manipulation_transform(...)["transformations"][0]["transformation"] (a nested list)."""
    moves = list(moves)
    if len(moves) > limit:
        raise ValueError("edit: at most %d moves are supported, got %d" % (limit, len(moves)))
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


def move_copies(copies, m):
    """copies (None, a bool, or one bool per move, like rest) -> [bool] of m: True where the move is a copy (DESIGN.md, "Copying
    objects"), which takes as the move would and leaves its source in place."""
    if copies is None:
        return [False] * m
    flags = [copies] * m if isinstance(copies, (bool, np.bool_)) else list(copies) if hasattr(copies, "__iter__") else None
    if flags is None or len(flags) != m or any(not isinstance(c, (bool, np.bool_)) for c in flags):
        raise ValueError("copies must be None, True / False, or one of them for each of the %d moves, got %r" % (m, copies))
    return [bool(c) for c in flags]


def _check_copies(copies, mv, drops, ordered=True, sets=None):
    """The copy flags of moves with labels mv and rest drops `drops`, checked -> [bool]: no copy drops the rest of its label (it
    vacates nothing) and, when the moves apply in order, no move of a label follows a copy of it (its vacate would erase the copy,
    which carries the label).  sets (move_groups; None: each move's own label): a move whose set holds a label of an earlier
    copy's set follows a copy of that label."""
    flags = move_copies(copies, len(mv))
    sets = sets or [(k,) for k in mv]
    for i, (c, d) in enumerate(zip(flags, drops)):
        if c and d:
            raise ValueError("copy: move %d: a copy cannot drop the rest of its label (rest 'drop'): it vacates nothing" % i)
        if ordered and not c:
            for j in range(i):
                shared = sorted(set(sets[j]) & set(sets[i])) if flags[j] else []
                if shared:
                    raise ValueError("copy: move %d of label %d follows copy %d of that label (its vacate would erase the copy)"
                                     % (i, shared[0], j))
    return flags


def _copy_flags(flags):
    """The HOST int32 copy flags of the _copies entry points."""
    return (C.c_int32 * len(flags))(*[int(c) for c in flags])


def move_groups(groups, mv, ins_num, who="group"):
    """groups (None, or one entry per move: None or an iterable of labels) -> one sorted tuple of labels per move, or None when
    every entry is None (DESIGN.md, "Moving objects together").  A move's set G moves every label of G as one rigid body; it must
    hold the move's label, and its labels lie in [0, ins_num].  An entry None is the move's own label."""
    if groups is None:
        return None
    if isinstance(groups, (str, bytes, dict)) or not hasattr(groups, "__iter__"):
        raise ValueError("%s: groups must be None or one entry per move, got %r" % (who, groups))
    groups = list(groups)
    if len(groups) != len(mv):
        raise ValueError("%s: groups must be None or one entry per move (%d), got %d" % (who, len(mv), len(groups)))
    if all(g is None for g in groups):
        return None
    out = []
    for i, (g, label) in enumerate(zip(groups, mv)):
        if g is None:
            out.append((label,))
            continue
        if isinstance(g, (str, bytes, dict)) or not hasattr(g, "__iter__"):
            raise ValueError("%s: move %d: a group must be None or an iterable of labels, got %r" % (who, i, g))
        ks = sorted(set(_labels(list(g), ins_num, who)))
        if label not in ks:
            raise ValueError("%s: move %d: the group %s does not hold the moved label %d" % (who, i, ks, label))
        out.append(tuple(ks))
    return out


def _group_words(sets):
    """The HOST uint32 [n][4] label words of the _groups entry points."""
    words = [w for ks in sets for w in label_words(ks)]
    return (C.c_uint32 * len(words))(*words)


def _group_mask(occ, labels, ks, level, piece, scene_transform, extents):
    """bool grid: the solid points of the labels ks, each label the piece applies to cut by the piece (region_drops)."""
    mask = torch.zeros_like(labels, dtype=torch.bool)
    keep = None
    applies = None if piece is None else label_words(range(MAX_LABELS)) if piece.applies is None else piece.applies
    for k in ks:
        mk = labels == int(k)
        if applies is not None and (applies[k >> 5] >> (k & 31)) & 1:
            if keep is None:
                keep = _region_keeps(piece, scene_transform, occ.shape[0], extents, occ.device)
            mk &= keep
        mask |= mk
    return mask & (occ > level)


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
    return _mask_box(mask, margin)


def _mask_box(mask, margin):
    """solid_box of the points of a bool grid."""
    if not bool(mask.any()):
        return EMPTY_BOX
    dim = mask.shape[0]
    box = []
    for a in range(3):
        idx = torch.nonzero(mask.any(dim=tuple(c for c in range(3) if c != a))).flatten()
        box += [max(int(idx[0]) - int(margin), 0), min(int(idx[-1]) + int(margin), dim - 1)]
    return tuple(box)


# ----------------------------------------------------------------------------------------------------------------- deformations
# DESIGN.md, "Deforming objects": a move bends, twists and tapers its object where it stands, before the move.
MAX_KNOTS = 64


def _det_interval_min(A, B):
    """The minimum over s in [0, 1] of det(A + s (B - A)) for 2x2 row-major A, B, in the library's operation order."""
    D = [B[0] - A[0], B[1] - A[1], B[2] - A[2], B[3] - A[3]]
    d0, a2 = A[0] * A[3] - A[1] * A[2], D[0] * D[3] - D[1] * D[2]
    b1 = ((A[0] * D[3] + D[0] * A[3]) - A[1] * D[2]) - D[1] * A[2]
    lo = min(d0, (d0 + b1) + a2)
    if a2 > 0.0:
        s = -b1 / (2.0 * a2)
        if 0.0 < s < 1.0:
            lo = min(lo, d0 - (b1 * b1) / (4.0 * a2))
    return lo


def deformation_problem(frame, h0, dh, knots):
    """The library's checks of a deformation (frame [12]: e_u, e_v, e_h, c; knots [K, 6]: A row-major, then t) in its order ->
    the reason it is rejected, or None."""
    frame = [float(v) for v in np.asarray(frame, dtype=np.float64).reshape(-1)]
    knots = np.asarray(knots, dtype=np.float64).reshape(-1, 6)
    K = knots.shape[0]
    if not 2 <= K <= MAX_KNOTS:
        return "n_knots %d is not 0 and outside [2, %d]" % (K, MAX_KNOTS)
    if not (np.isfinite(frame).all() and np.isfinite(knots).all() and np.isfinite(h0) and np.isfinite(dh)):
        return "a value is not finite"
    if not dh > 0.0:
        return "dh %g must be > 0" % dh
    e = frame
    ok = all(abs(((e[3 * a] * e[3 * b] + e[3 * a + 1] * e[3 * b + 1]) + e[3 * a + 2] * e[3 * b + 2]) - (1.0 if a == b else 0.0))
             <= 1e-9 for a in range(3) for b in range(3))
    for a in range(3):
        a1, a2 = (a + 1) % 3, (a + 2) % 3
        ok = ok and abs((e[a1] * e[3 + a2] - e[a2] * e[3 + a1]) - e[6 + a]) <= 1e-9
    if not ok:
        return "the frame is not orthonormal and right-handed"
    for k in range(K - 1):
        if not _det_interval_min([float(v) for v in knots[k, :4]], [float(v) for v in knots[k + 1, :4]]) > 0.0:
            return "det A(h) <= 0 on knot interval %d" % k
    return None


class Deformation:
    """A checked deformation of a move's object (DESIGN.md, "Deforming objects"): in the frame of centre `centre`, up axis `up`
    (e_h) and forward axis `forward` (e_u; e_v = up x forward), the object's horizontal section at frame height h maps as
    (u, v) -> A(h) (u, v) + t(h), h kept.  A [K, 2, 2] and t [K, 2] are the knots at heights h0 + k dh (dh > 0, K in [2, 64]),
    interpolated linearly and clamped to the end knots.  ValueError with the library's message for a table it rejects: a
    non-finite value, dh <= 0, axes that are not orthonormal to 1e-9, or det A(h) <= 0 anywhere between the knots.
    Immutable; deformation() builds one from twist, bend and taper profiles."""
    __slots__ = ("frame", "h0", "dh", "knots", "_abi")

    def __init__(self, centre, up, forward, h0, dh, A, t):
        up, forward = np.asarray(up, dtype=np.float64).reshape(3), np.asarray(forward, dtype=np.float64).reshape(3)
        frame = np.concatenate([forward, np.cross(up, forward), up, np.asarray(centre, dtype=np.float64).reshape(3)])
        A, t = np.asarray(A, dtype=np.float64), np.asarray(t, dtype=np.float64)
        if A.ndim != 3 or A.shape[1:] != (2, 2) or t.shape != (A.shape[0], 2):
            raise ValueError("deformation: A must be [K, 2, 2] and t [K, 2], got shapes %s and %s" % (A.shape, t.shape))
        knots = np.concatenate([A.reshape(-1, 4), t], 1)
        why = deformation_problem(frame, float(h0), float(dh), knots)
        if why is not None:
            raise ValueError("deformation: " + why)
        d = _lib.Deformation()
        held = (C.c_double * knots.size)(*knots.reshape(-1).tolist())
        d.n_knots, d.h0, d.dh, d.knots = knots.shape[0], float(h0), float(dh), C.cast(held, C.POINTER(C.c_double))
        d.frame[:] = frame.tolist()
        for k, v in zip(self.__slots__, (frame, float(h0), float(dh), knots, (d, held))):
            object.__setattr__(self, k, v)
        frame.setflags(write=False)
        knots.setflags(write=False)

    def __setattr__(self, key, value):
        raise AttributeError("Deformation is immutable")

    def abi(self):
        """The dmnerf_deformation of this table (its knots held by this value)."""
        return self._abi[0]


def _profile(values, knots, what):
    if values is None:
        return None
    s = np.linspace(0.0, 1.0, knots)
    v = np.asarray([values(x) for x in s] if callable(values) else values, dtype=np.float64).reshape(-1)
    if v.shape != (knots,) or not np.isfinite(v).all():
        raise ValueError("deformation: %s must be %d finite values or a callable of the normalised height, got %d" % (what, knots,
                                                                                                               v.size))
    return v


def deformation(centre, up, h0, h1, knots=33, twist=None, bend=None, bend_dir=None, taper=None):
    """The Deformation that twists, bends and tapers an object standing at `centre` along `up` between frame heights h0 < h1
    (heights along up, from the centre).  Each profile is `knots` values or a callable of the normalised height in [0, 1]:
    twist, an angle in degrees about up; bend, an offset along the horizontal direction bend_dir; taper, a horizontal scale
    (each > 0).  Per knot A = R(twist) diag(taper, taper) and t = (bend, 0); e_u is bend_dir (made horizontal) with a bend and
    otherwise a horizontal axis.  cos / sin are numpy's."""
    knots = int(knots)
    if not 2 <= knots <= MAX_KNOTS:
        raise ValueError("deformation: n_knots %d is not 0 and outside [2, %d]" % (knots, MAX_KNOTS))
    if not (np.isfinite([h0, h1]).all() and h1 > h0):
        raise ValueError("deformation: the height range [%r, %r] must be finite and h1 > h0" % (h0, h1))
    up = np.asarray(up, dtype=np.float64).reshape(3)
    if not (np.isfinite(up).all() and np.linalg.norm(up) > 0):
        raise ValueError("deformation: up must be a finite non-zero vector")
    up = up / np.linalg.norm(up)
    tw, bd, tp = _profile(twist, knots, "twist"), _profile(bend, knots, "bend"), _profile(taper, knots, "taper")
    if bd is not None:
        if bend_dir is None:
            raise ValueError("deformation: a bend needs bend_dir")
        e = np.asarray(bend_dir, dtype=np.float64).reshape(3)
        e = e - np.dot(e, up) * up
        if not np.linalg.norm(e) > 1e-9:
            raise ValueError("deformation: bend_dir must not be parallel to up")
    else:
        e = np.eye(3)[int(np.argmin(np.abs(up)))]
        e = e - np.dot(e, up) * up
    e = e / np.linalg.norm(e)
    if tp is not None and not (tp > 0).all():
        raise ValueError("deformation: taper must be > 0")
    th = np.radians(tw) if tw is not None else np.zeros(knots)
    sc = tp if tp is not None else np.ones(knots)
    c, s = np.cos(th), np.sin(th)
    A = np.stack([np.stack([c * sc, -s * sc], -1), np.stack([s * sc, c * sc], -1)], 1)
    t = np.stack([bd if bd is not None else np.zeros(knots), np.zeros(knots)], -1)
    return Deformation(centre, up, e, float(h0), (float(h1) - float(h0)) / (knots - 1), A, t)


def move_deformations(deformations, m):
    """deformations (None, or one Deformation-or-None per move) -> a list of m, or None when every move is rigid."""
    if deformations is None:
        return None
    if isinstance(deformations, Deformation) or not hasattr(deformations, "__iter__"):
        raise ValueError("deformations must be None or one Deformation (or None) per move, got %r" % (deformations,))
    defs = list(deformations)
    if len(defs) != m or any(d is not None and not isinstance(d, Deformation) for d in defs):
        raise ValueError("deformations must be None or one Deformation (or None) for each of the %d moves" % m)
    return defs if any(d is not None for d in defs) else None


def _deformation_array(defs):
    """The HOST dmnerf_deformation [n] of the _deformed entry points (a rigid move: n_knots 0)."""
    arr = (_lib.Deformation * len(defs))()
    for i, d in enumerate(defs):
        if d is not None:
            arr[i] = d.abi()
    return arr


def edit_occupancy(model_fine, scene_transform, occ, labels, moves, boxes, extents=None, level=0.45, near=4.0, far=15.0,
                   N_importance=128, pieces=None, rest="keep", slab=0, copies=None, groups=None, deformations=None):
    """dmnerf_mesh_occupancy_edit: the moves [(label, 4x4)] applied in order, in place, to occ / labels ([dim]^3 float32 /
    int16 on the device: the keep-all sweep of model_fine on this grid), the network evaluated only at the target points
    inside each move's box (boxes: [m, 6] inclusive index boxes, EMPTY_BOX for none).  pieces / rest: as manipulator.  copies
    (None, a bool or one per move): the moves that are copies, which take as the move would and never vacate
    (dmnerf_mesh_occupancy_edit_copies; DESIGN.md, "Copying objects").  groups (None, or per move None or labels; DESIGN.md,
    "Moving objects together"): the labels each move carries as one body (dmnerf_mesh_occupancy_edit_groups).  deformations (None,
    or one Deformation or None per move; DESIGN.md, "Deforming objects"): each deformed move bends, twists or tapers its object
    (dmnerf_mesh_occupancy_edit_deformed).  Returns the number of target points evaluated."""
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
    sets = move_groups(groups, mv, ins_num)
    flags = _check_copies(copies, mv, drops, sets=sets)
    defs = move_deformations(deformations, len(mv))
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
    head = (ctx.handle, slot, _lib.doubles(T, 16), _lib.doubles(ext, 3), dim, (far - near) / N_importance, level, int(slab), descs)
    tail = (len(mv), _lib.ptr(occ), _lib.ptr(labels, torch.int16), C.byref(n))
    with torch.no_grad():
        if defs is not None:
            ctx.call("dmnerf_mesh_occupancy_edit_deformed", *head, _copy_flags(flags), None if sets is None else _group_words(sets),
                     _deformation_array(defs), *tail)
        elif sets is not None:
            ctx.call("dmnerf_mesh_occupancy_edit_groups", *head, _copy_flags(flags), _group_words(sets), *tail)
        elif any(flags):
            ctx.call("dmnerf_mesh_occupancy_edit_copies", *head, _copy_flags(flags), *tail)
        else:
            ctx.call("dmnerf_mesh_occupancy_edit", *head, *tail)
    return int(n.value)


def edit_boxes(occ, labels, moves, scene_transform, extents=None, level=0.45, margin=2, pieces=None, groups=None):
    """The default boxes of edited_sweep from the unedited sweep: per move, solid_box of its label's solid points (those its
    piece keeps, with a piece) grown by margin -> int [m, 6].  groups (as edited_sweep): a group's box holds the solid points of
    every label of its set, the piece applied to the labels it applies to."""
    if int(margin) != margin or int(margin) < 0:
        raise ValueError("edit: margin must be an integer >= 0, got %r" % (margin,))
    mv = [int(m[0]) for m in moves]
    regions = list(pieces) if pieces is not None else [None] * len(mv)
    sets = move_groups(groups, mv, MAX_LABELS - 1) or [(k,) for k in mv]
    dim = occ.shape[0]
    out = []
    for k, r, ks in zip(mv, regions, sets):
        if len(ks) > 1:
            out.append(_mask_box(_group_mask(occ, labels, ks, level, r, scene_transform, extents), int(margin)))
            continue
        keep = None if r is None else _region_keeps(r, scene_transform, dim, extents, occ.device)
        out.append(solid_box(occ, labels, k, level, int(margin), keep))
        del keep
    return np.asarray(out, dtype=np.int64).reshape(len(mv), 6)


def edited_sweep(model_fine, scene_transform, moves, grid_dim=256, extents=None, level=0.45, near=4.0, far=15.0, N_importance=128,
                 margin=2, boxes=None, pieces=None, rest="keep", copies=None, groups=None, deformations=None):
    """The labelled sweep of the edited scene -> (occ [dim]^3 float32, labels [dim]^3 int16) on the device: the keep-all sweep of
    model_fine (occupancy_objects), then the moves [(label, 4x4 in the network frame, as manipulator_eval's transformation)]
    applied in order (edit_occupancy).  A move shows at p what the network holds at trans p, as rigid_rays renders it: the
    object lands at inv(trans) x.  boxes: per move the index box of the target points evaluated; by default the box of the
    moved label's solid points in the unedited grid (of those its piece keeps, with a piece) grown by `margin` voxels.
    pieces / rest: as manipulator (a Region or None per move; "keep" / "drop", or one per move).  copies (None, a bool or one
    per move; DESIGN.md, "Copying objects"): a copy takes as its move would and leaves the source in place; the copy keeps the
    source's label: a second connected piece of it where it does not touch its source, one piece with it where it does.
    groups (None, or one entry per move: None or an iterable of labels holding the move's label; DESIGN.md, "Moving objects
    together"): each move carries every label of its set as one rigid body -- a table with what stands on it -- in one pass;
    a target of any label of the set is taken with its own label, and every label of the set is vacated.  The default box holds
    the whole set.  carried_labels finds the set of what rests on an object.  deformations (None, or one Deformation or None per
    move; DESIGN.md, "Deforming objects"): a deformed move bends, twists or tapers its object where it stands, before the move; the
    default box is still the source's."""
    from .manipulator import move_pieces, move_rests
    from .mesh import check_transform
    T = check_transform(scene_transform)
    dev = next(model_fine.parameters()).device
    ins_num = int(model_fine.ins_linear.weight.shape[0]) - 1
    mv, _ = _check_moves(moves, ins_num)
    level = _check_level(level)
    _check_copies(copies, mv, move_rests(rest, len(mv)), sets=move_groups(groups, mv, ins_num))
    move_deformations(deformations, len(mv))
    move_pieces(pieces, mv, ins_num, dev)
    if int(margin) != margin or int(margin) < 0:
        raise ValueError("edit: margin must be an integer >= 0, got %r" % (margin,))
    if boxes is not None:
        boxes = _check_boxes(boxes, len(mv), int(grid_dim))
    with torch.no_grad():
        occ, labels = occupancy_objects(model_fine, T, object_mask(ins_num, remove=[]), grid_dim, extents, near, far, N_importance,
                                        device=dev)
        if boxes is None:
            boxes = edit_boxes(occ, labels, moves, T, extents, level, margin, pieces, groups)
        edit_occupancy(model_fine, T, occ, labels, moves, boxes, extents, level, near, far, N_importance, pieces, rest, copies=copies,
                       groups=groups, deformations=deformations)
    return occ, labels


def edited_mesh(model_fine, scene_transform, moves, grid_dim=256, extents=None, level=0.45, near=4.0, far=15.0, N_importance=128,
                margin=2, boxes=None, pieces=None, rest="keep", min_cluster=400, per_object=False, copies=None, groups=None,
                deformations=None):
    """The mesh of an edited scene: edited_sweep (same arguments) -> marching cubes -> scene space -> normals -> small-cluster
    removal.  Returns extract_mesh's keys as device tensors -- vertices, triangles, normals, clean_vertices, clean_normals,
    clean_triangles -- and labels (int64 per clean vertex: mesh.vertex_labels of its index-space vertex, the label of the
    inside end of its edge, from the edited grid; no label rays are rendered).  per_object: also objects, the
    meshes_from_labelled_grid of the edited grid for every label with solid points except ins_num.  copies, groups, deformations:
    as edited_sweep."""
    from .mesh import EXTENTS, check_transform, clean_mesh, marching_cubes, to_scene, vertex_labels, vertex_normals
    T = check_transform(scene_transform)
    ext = EXTENTS if extents is None else extents
    ins_num = int(model_fine.ins_linear.weight.shape[0]) - 1
    with torch.no_grad():
        occ, labels = edited_sweep(model_fine, T, moves, grid_dim, ext, level, near, far, N_importance, margin, boxes, pieces, rest,
                                   copies=copies, groups=groups, deformations=deformations)
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


# ----------------------------------------------------------------------------------------------------------------- moved renders
# DESIGN.md, "Rendering moved objects": edited_sweep's moves applied per render sample, inside the stage render, so that a render
# and a mesh of one edit agree.  render_rays(moves=) and render_frame(moves=) take the value render_moves returns.
class MovedScene:
    """Checked moves for render_rays(moves=) / render_frame(moves=): the dmnerf_render_moves the library reads, and the move
    descriptions and region bits it points into, held for as long as the value lives.  copies: per move, whether it is a copy
    (DESIGN.md, "Copying objects"); groups: per move, the labels it carries (DESIGN.md, "Moving objects together");
    deformations: per move, its Deformation or None (DESIGN.md, "Deforming objects").  Immutable."""
    __slots__ = ("_desc", "_held", "device", "labels", "boxes", "rest_drop", "level", "voxel", "copies", "_flags", "groups", "_words",
                 "deformations", "_defs")

    def __init__(self, desc, held, device, labels, boxes, rest_drop, level, voxel, copies=None, groups=None, deformations=None):
        copies = tuple(bool(c) for c in copies) if copies is not None else (False,) * len(labels)
        sets = tuple(tuple(g) for g in groups) if groups is not None else tuple((k,) for k in labels)
        defs = tuple(deformations) if deformations is not None else (None,) * len(labels)
        for k, v in zip(self.__slots__, (desc, held, device, labels, tuple(map(tuple, boxes.tolist())), tuple(rest_drop), level,
                                         voxel, copies, _copy_flags(copies) if any(copies) else None, sets,
                                         _group_words(sets) if groups is not None else None, defs,
                                         _deformation_array(defs) if any(d is not None for d in defs) else None)):
            object.__setattr__(self, k, v)

    def __setattr__(self, key, value):
        raise AttributeError("MovedScene is immutable")

    def abi(self):
        """The dmnerf_render_moves of these moves."""
        return self._desc

    def copy_flags(self):
        """The copy flags dmnerf_render_moved_copies reads (HOST int32 [n_moves]), or None when no move is a copy."""
        return self._flags

    def group_words(self):
        """The label sets dmnerf_render_moved_groups reads (HOST uint32 [n_moves][4]), or None when no group was given."""
        return self._words

    def deformation_array(self):
        """The deformations dmnerf_render_moved_deformed reads (HOST dmnerf_deformation [n_moves]), or None when every move is
        rigid."""
        return self._defs


def render_moves(occ, labels, scene_transform, moves, extents=None, level=0.45, near=4.0, far=15.0, N_importance=128, margin=2,
                 boxes=None, pieces=None, rest="keep", copies=None, groups=None, deformations=None):
    """The moves [(label, 4x4 in the network frame)] of edited_sweep, checked for the moved render -> a MovedScene.  occ / labels:
    the unedited keep-all sweep ([dim]^3 float32 / int16 on the device) that the default boxes come from (edit_boxes, as
    edited_sweep) and whose grid (scene_transform, extents, dim) the boxes index.  level, margin, boxes, pieces, rest: as
    edited_sweep; the voxel of the occupancy test is the sweep's (far - near) / N_importance.  moves, pieces and rest may be
    arrange_objects' moves, pieces and rest unchanged, or manipulator_eval's [(label, 4x4)].  Labels are checked against the
    networks when the render runs.  copies, groups: as edited_sweep (arrange_objects' copies and groups unchanged).
    deformations: as edited_sweep; a deformed move's view directions are its pulled-back ray tangents."""
    from .manipulator import move_pieces, move_rests
    from .mesh import EXTENTS, check_transform
    T = check_transform(scene_transform)
    ext = EXTENTS if extents is None else extents
    mv, mats = _check_moves(moves, MAX_LABELS - 1)
    if not mv:
        raise ValueError("render_moves: give between 1 and %d moves" % _lib.MAX_MOVES)
    level = _check_level(level)
    drops = move_rests(rest, len(mv))
    sets = move_groups(groups, mv, MAX_LABELS - 1)
    flags = _check_copies(copies, mv, drops, sets=sets)
    defs = move_deformations(deformations, len(mv))
    if int(margin) != margin or int(margin) < 0:
        raise ValueError("edit: margin must be an integer >= 0, got %r" % (margin,))
    with np.errstate(divide="ignore", invalid="ignore"):
        voxel = np.float32(np.float64(far - near) / np.float64(N_importance))
    if not (np.isfinite(voxel) and voxel > 0):
        raise ValueError("render_moves: the voxel (far - near) / N_importance = %r must be finite and > 0" % (float(voxel),))
    if boxes is not None:
        boxes = _check_boxes(boxes, len(mv), occ.shape[0])
    regions = move_pieces(pieces, mv, MAX_LABELS - 1, occ.device) or [None] * len(mv)
    dim = _check_sweep(occ, labels, "render_moves")
    if boxes is None:
        boxes = _check_boxes(edit_boxes(occ, labels, moves, T, ext, level, margin, pieces, sets), len(mv), dim)
    descs = _edit_moves(mv, mats, boxes, drops, regions, occ.device)
    d = _lib.RenderMoves()
    d.moves, d.n_moves, d.dim = C.cast(descs, C.POINTER(_lib.EditMove)), len(mv), dim
    d.transform[:] = np.asarray(T, dtype=np.float64).reshape(-1).tolist()
    d.extents[:] = np.asarray(ext, dtype=np.float64).reshape(-1).tolist()
    d.level, d.voxel = level, float(voxel)
    return MovedScene(d, (descs, [r.bits for r in regions if r is not None]), occ.device, tuple(mv), boxes, drops, level,
                      float(voxel), flags, sets, defs)


# ----------------------------------------------------------------------------------------------------------------- collisions
# DESIGN.md, "Collision checks": grid-only checks of moves on the labelled keep-all sweep (edited_sweep's), each candidate on its
# own.  The moved object at p is the unedited grid at the nearest grid index of trans p, as edited_sweep samples it on an exact
# grid; off the grid points it is the sweep resampled at its own resolution, not the network at trans p.
ALL_LABELS = [0xFFFFFFFF] * 4


def _voxel_volume(T, ext, dim):
    return abs(np.linalg.det(T[:3, :3])) * float(np.prod(np.asarray(ext, dtype=np.float64) / (dim - 1)))


def _check_sweep(occ, labels, who):
    dim = _check_grid(occ, labels, who)
    if labels is None or labels.dtype != torch.int16 or occ.dtype != torch.float32:
        raise ValueError("%s: occ must be float32 and labels int16" % who)
    return dim


def move_overlap(occ, labels, scene_transform, moves, extents=None, level=0.45, boxes=None, margin=2, pieces=None, rest="keep",
                 obstacles=None, copies=None, groups=None, deformations=None):
    """dmnerf_move_overlap: each move [(label, 4x4 in the network frame)] checked on its own against the labelled keep-all sweep
    occ / labels ([dim]^3 float32 / int16 on the device; an edited_sweep result is accepted unchanged).  boxes, margin, pieces,
    rest: as edited_sweep (default boxes: edit_boxes).  obstacles: the labels that count as obstacles (default every label).
    Returns one dict per move: label, landed (the voxels the moved object occupies after the move), overlap {label: voxels}
    (labels with voxels > 0: solid obstacle points the moved object lands on; the points the move vacates are not obstacles),
    overlap_volume {label: voxels times the inventory's voxel volume} and total (the overlapping voxels).  copies (None, a bool or
    one per move; DESIGN.md, "Copying objects"): a copy vacates nothing, so its own label's solid points are obstacles too.
    groups (as edited_sweep; DESIGN.md, "Moving objects together"): each candidate moves its whole set; landed and overlap count
    every label of the set, and the points the set vacates are not obstacles (a copy's stay).  deformations (as edited_sweep;
    DESIGN.md, "Deforming objects"): each candidate's object is deformed before its move."""
    from .manipulator import move_pieces, move_rests
    from .mesh import EXTENTS, check_transform
    T = check_transform(scene_transform)
    dim = _check_sweep(occ, labels, "move_overlap")
    ext = EXTENTS if extents is None else extents
    ins_num = MAX_LABELS - 1
    mv, mats = _check_moves(moves, ins_num, _lib.MAX_CANDIDATES)
    level = _check_level(level)
    drops = move_rests(rest, len(mv))
    sets = move_groups(groups, mv, ins_num)
    flags = _check_copies(copies, mv, drops, ordered=False)
    defs = move_deformations(deformations, len(mv))
    regions = move_pieces(pieces, mv, ins_num, occ.device) or [None] * len(mv)
    words = ALL_LABELS if obstacles is None else label_words(obstacles)
    if not mv:
        return []
    if boxes is None:
        boxes = edit_boxes(occ, labels, moves, T, ext, level, margin, pieces, sets)
    boxes = _check_boxes(boxes, len(mv), dim)
    descs = _edit_moves(mv, mats, boxes, drops, regions, occ.device)
    overlap = np.zeros((len(mv), MAX_LABELS), dtype=np.int64)
    landed = np.zeros(len(mv), dtype=np.int64)
    ctx = get_context(occ.device)
    head = (ctx.handle, _lib.ptr(occ), _lib.ptr(labels, torch.int16), dim, level, _lib.doubles(T, 16), _lib.doubles(ext, 3), descs)
    tail = (len(mv), (C.c_uint32 * 4)(*words), overlap.ctypes.data_as(C.POINTER(C.c_int64)), landed.ctypes.data_as(C.POINTER(C.c_int64)))
    if defs is not None:
        ctx.call("dmnerf_move_overlap_deformed", *head, _copy_flags(flags), None if sets is None else _group_words(sets),
                 _deformation_array(defs), *tail)
    elif sets is not None:
        ctx.call("dmnerf_move_overlap_groups", *head, _copy_flags(flags), _group_words(sets), *tail)
    elif any(flags):
        ctx.call("dmnerf_move_overlap_copies", *head, _copy_flags(flags), *tail)
    else:
        ctx.call("dmnerf_move_overlap", *head, *tail)
    unit = _voxel_volume(T, ext, dim)
    return [_count_report(mv[i], landed[i], overlap[i], unit, "overlap") for i in range(len(mv))]


def _edit_moves(mv, mats, boxes, drops, regions, device):
    """The ABI moves (dmnerf_edit_move) of checked labels, 4x4 matrices, boxes, rest drops and pieces (labels up to 127)."""
    from .manipulator import _piece_region
    descs = (_lib.EditMove * len(mv))()
    for i in range(len(mv)):
        d = descs[i]
        d.label, d.rest_drop = mv[i], int(drops[i])
        d.trans[:] = mats[i][:3].reshape(-1).tolist()
        d.box[:] = [int(v) for v in boxes[i]]
        d.piece = _piece_region(regions[i], mv[i], MAX_LABELS - 1, device)
    return descs


def _count_report(label, landed, counts, unit, key):
    """One move's counts as move_overlap and edited_grid report them: label, landed, key {label: voxels} (labels with voxels > 0),
    key_volume {label: voxels times the voxel volume `unit`} and total."""
    hit = {int(k): int(counts[k]) for k in np.nonzero(counts)[0]}
    return {"label": label, "landed": int(landed), key: hit, key + "_volume": {k: v * unit for k, v in hit.items()},
            "total": int(counts.sum())}


def _translate(v):
    m = np.eye(4)
    m[:3, 3] = v
    return m


def slide_steps(direction, max_distance, step, base=None):
    """The candidates of slide_until_contact -> (unit direction, distances s_k, 4x4 moves base @ translate(-s_k d)).  s_k =
    k step for k = 0 .. K - 1, the last one max_distance itself; ValueError for more than MAX_CANDIDATES steps."""
    d = np.asarray(direction, dtype=np.float64).reshape(-1)
    if d.shape != (3,) or not np.isfinite(d).all() or not np.linalg.norm(d) > 0:
        raise ValueError("slide: direction must be 3 finite numbers, not all 0, got %r" % (d.tolist(),))
    d = d / np.linalg.norm(d)
    max_distance, step = float(max_distance), float(step)
    if not (np.isfinite(max_distance) and max_distance >= 0):
        raise ValueError("slide: max_distance must be finite and >= 0, got %r" % max_distance)
    if not (np.isfinite(step) and step > 0):
        raise ValueError("slide: step must be finite and > 0, got %r" % step)
    n = int(np.ceil(max_distance / step)) + 1
    if n > _lib.MAX_CANDIDATES:
        raise ValueError("slide: %d steps of %g to %g exceed the %d candidates of one check" % (n, step, max_distance,
                                                                                              _lib.MAX_CANDIDATES))
    base = np.eye(4) if base is None else _move_matrix(base, 0)
    s = np.minimum(np.arange(n, dtype=np.float64) * step, max_distance)
    return d, s, [base @ _translate(-sk * d) for sk in s]


def slide_result(d, steps, results, tolerance, base=None):
    """The answer of slide_until_contact from the move_overlap results of its steps."""
    base = np.eye(4) if base is None else np.asarray(base, dtype=np.float64)
    profile = [r["total"] for r in results]
    first = next((k for k, v in enumerate(profile) if v > tolerance), None)
    if first is None:
        distance, contact = float(steps[-1]), None
    else:
        contact = {"distance": float(steps[first]), "overlap": results[first]["overlap"]}
        distance = float(steps[first - 1]) if first > 0 else None
    trans = None if distance is None else (base @ _translate(-distance * d)).tolist()
    return {"distance": distance, "transformation": trans, "contact": contact, "steps": [float(v) for v in steps],
            "profile": profile}


def slide_until_contact(occ, labels, scene_transform, label, direction, max_distance, step=None, base=None, tolerance=0,
                        extents=None, level=0.45, margin=2, piece=None, rest="keep", obstacles=None):
    """How far object `label` (or its piece) can slide along `direction` (network frame) before it overlaps an obstacle of the
    sweep occ / labels by more than `tolerance` voxels.  The candidates base @ translate(-s_k d) (d the unit direction): the
    object moved by base (it lands at inv(base) x), then shifted by s_k d, s_k = k step up to max_distance (step: default the
    smallest grid spacing), all checked in one move_overlap call (at most MAX_CANDIDATES steps).  Returns
      distance:       the largest s_k before the first step that overlaps, max_distance without contact, None when base
                      itself overlaps;
      transformation: the 4x4 (nested list) at that distance, as rigid_rays, manipulator_eval and edited_sweep take it;
      contact:        None, or {distance, overlap} of the first overlapping step;
      steps, profile: every s_k and its total overlap.
    The object is checked at the steps only: an obstacle thinner than one step can be passed through."""
    from .mesh import EXTENTS, check_transform
    T = check_transform(scene_transform)
    ext = EXTENTS if extents is None else extents
    if int(tolerance) != tolerance or int(tolerance) < 0:
        raise ValueError("slide: tolerance must be an integer >= 0 voxels, got %r" % (tolerance,))
    if step is None:
        A, _ = grid_affine(T, occ.shape[0], ext)
        step = float(np.linalg.norm(A, axis=0).min())
    d, s, mats = slide_steps(direction, max_distance, step, base)
    pieces = None if piece is None else [piece]
    box = edit_boxes(occ, labels, [(label, mats[0])], T, ext, _check_level(level), margin, pieces)[0]
    results = move_overlap(occ, labels, T, [(label, m) for m in mats], ext, level, [box] * len(mats), margin,
                           None if piece is None else [piece] * len(mats), rest, obstacles)
    return slide_result(d, s, results, int(tolerance), mats[0])


def object_contacts(occ, labels, scene_transform, extents=None, level=0.45):
    """dmnerf_object_contacts: which objects of a labelled sweep touch.  Returns faces int64 [3, 128, 128] (faces[a, l1, l2]:
    the solid points of l1 whose +a index neighbour is a solid point of l2 != l1), axes [3, 3] (the unit network-frame direction
    of each index axis) and face_area [3] (the network-frame area of one voxel face across each axis)."""
    from .mesh import EXTENTS, check_transform
    T = check_transform(scene_transform)
    dim = _check_sweep(occ, labels, "object_contacts")
    ext = EXTENTS if extents is None else extents
    level = _check_level(level)
    faces = np.zeros((3, MAX_LABELS, MAX_LABELS), dtype=np.int64)
    ctx = get_context(occ.device)
    ctx.call("dmnerf_object_contacts", ctx.handle, _lib.ptr(occ), _lib.ptr(labels, torch.int16), dim, level, MAX_LABELS,
             faces.ctypes.data_as(C.POINTER(C.c_int64)))
    return contacts_from_faces(faces, T, dim, ext)


def contacts_from_faces(faces, scene_transform, dim, extents=None):
    """object_contacts' dict from its face counts and the grid."""
    A, _ = grid_affine(scene_transform, dim, extents)
    area = [float(np.linalg.norm(np.cross(A[:, (a + 1) % 3], A[:, (a + 2) % 3]))) for a in range(3)]
    return {"faces": faces, "axes": (A / np.linalg.norm(A, axis=0)).T.copy(), "face_area": np.array(area)}


def carried_labels(occ, labels, scene_transform, label, down, extents=None, level=0.45, min_faces=1, exclude=()):
    """What rests on object `label`, transitively (DESIGN.md, "Moving objects together"): the labels whose solid points lie on
    those of `label` along the down axis (supports of object_contacts, pairs of at least min_faces faces), then what rests on
    those, and so on -> {"group": sorted labels with `label`, "chain": {label: (the label it rests on, faces)}}, the group=
    that moves the object with what it carries.  exclude: labels never added (a voxelised wall or floor can touch a table top
    from above); the chain says why each label was added.  Whole labels only: a caller that moves a piece of an object passes
    the group it wants explicitly."""
    label = _labels([label], MAX_LABELS - 1, "carried_labels")[0]
    exclude = set(_labels(exclude, MAX_LABELS - 1, "carried_labels"))
    return _carried(supports(object_contacts(occ, labels, scene_transform, extents, level), down, min_faces), label, exclude)


def _carried(on, label, exclude):
    """carried_labels' closure over a supports() result `on`: breadth first from `label`, ascending labels at each step."""
    group, chain, frontier = {label}, {}, [label]
    while frontier:
        base = frontier.pop(0)
        for top in sorted(on):
            if top in group or top in exclude:
                continue
            faces = dict(on[top]).get(base)
            if faces is not None:
                group.add(top)
                chain[top] = (base, faces)
                frontier.append(top)
    return {"group": sorted(group), "chain": chain}


def supports(contacts, down, min_faces=1):
    """Which object rests on which, from object_contacts: along the index axis closest to +-down (network frame), the labels
    below each label's solid points -> {label: [(label_below, faces), ...]}, most faces first (then ascending label); pairs
    with fewer than min_faces faces are left out."""
    a, sign = down_axis(contacts["axes"], down, "supports")
    if int(min_faces) != min_faces or int(min_faces) < 1:
        raise ValueError("supports: min_faces must be an integer >= 1, got %r" % (min_faces,))
    f = np.asarray(contacts["faces"])[a]
    if sign < 0:                                       # +e_a points up: the neighbour at p + e_a is above
        f = f.T
    out = {}
    for top, below in zip(*np.nonzero(f >= int(min_faces))):
        out.setdefault(int(top), []).append((int(below), int(f[top, below])))
    return {k: sorted(v, key=lambda x: (-x[1], x[0])) for k, v in sorted(out.items())}


def down_axis(axes, down, who):
    """The index axis closest to +-down (network frame), given the unit network-frame direction of each index axis as the rows
    of axes [3, 3] -> (axis, sign): sign +1 when +e_axis points down, -1 when it points up."""
    dn = np.asarray(down, dtype=np.float64).reshape(-1)
    if dn.shape != (3,) or not np.isfinite(dn).all() or not np.linalg.norm(dn) > 0:
        raise ValueError("%s: down must be 3 finite numbers, not all 0, got %r" % (who, dn.tolist()))
    dots = np.asarray(axes) @ (dn / np.linalg.norm(dn))
    a = int(np.argmax(np.abs(dots)))
    return a, (1 if dots[a] > 0 else -1)


# ----------------------------------------------------------------------------------------------------------------- placement
# DESIGN.md, "Object placement": where an object lowered along the down axis comes to rest at every horizontal offset of the
# labelled keep-all sweep, what holds it up and whether it stands; index space, integers.
PLACE_MAX_DIM = 1024                 # int16 heights in the column table


def _check_point(x, what):
    p = np.asarray(x, dtype=np.float64).reshape(-1)
    if p.shape != (3,) or not np.isfinite(p).all():
        raise ValueError("placement: %s must be 3 finite numbers, got %r" % (what, p.tolist()))
    return p


def placement_map(occ, labels, scene_transform, label, down, lift=0, extents=None, level=0.45, piece=None, rest="keep",
                  obstacles=None, base=None, box=None, scene=None, copy=False, group=None):
    """dmnerf_placement_map: object `label` (or its piece, with rest "keep" / "drop" as move_overlap) raised by `lift` voxels and
    lowered along the index axis closest to +-down (network frame, chosen as supports chooses it), at every horizontal offset
    that keeps it inside the grid of the labelled keep-all sweep occ / labels.  obstacles: the labels that count (default all).
    base (a 4x4 move in the network frame, as move_overlap takes it) places the object as that move leaves it instead
    (dmnerf_placement_maps; DESIGN.md, "Turned placements"): sampled from the grid through the source box `box` (default
    edit_boxes' box, margin 2), its points carried outside the grid lost.
    scene (DESIGN.md, "Arranging objects"): an (occ, labels) pair of the same shape, dtype and device, e.g. an edited_grid
    result; the object is still sampled from occ / labels, but the obstacles, the points it vacates and the labels it rests on
    come from the scene (dmnerf_placement_maps_in_scene; without a base, the identity base with the default box).
    copy (DESIGN.md, "Copying objects"): place a copy of the object, its source standing: the scene's solid points of the label
    stay obstacles.  A copy always takes the based path (the identity base with the default box without one) and the scene is
    occ / labels when none is given; rest must be "keep".
    group (None or labels holding `label`; DESIGN.md, "Moving objects together"): place the solid points of every label of the
    group (the piece applied to the labels it applies to) as one body, its default box the group's; what the group vacates is no
    obstacle, and a contact inside the group is never a support.  A group takes the based path as a copy does.
    Returns a dict:
      drop, support, contacts: device maps [U, V] (int32, int16, int32): the voxels it falls (-1: blocked where it is raised),
                      the obstacle label under most of its resting runs (-1: blocked, or resting on the grid's floor), and the
                      runs that rest on an obstacle;
      offset_lo:      the offset (u, v) of entry [0, 0], in voxels along the horizontal axes;
      axis, sign, horizontal: the down axis, +1 when +e_axis points down, and the two horizontal index axes (ascending);
      centre:         the object's exact centre of mass in index space (3 Fractions, axes i, j, k), from its runs;
      runs, points:   its vertical runs and its points;
      base, box:      the move (4x4, None without one) and its source box (None without a base);
      points_before:  the object's points before the move (points without a base): a difference is clipping or resampling;
    and what placement() needs to describe one offset."""
    if base is None and box is not None:
        raise ValueError("placement: box needs a base")
    if base is not None:
        base = _move_matrix(base, 0)
    if box is not None:
        box = _check_boxes([box], 1, occ.shape[0])[0]
    c = _placement_call(occ, labels, scene_transform, label, down, lift, extents, level, piece, rest, obstacles, scene, copy, group)
    if base is None and c["scene"] is not None:
        m, status = _placement_maps(c, [np.eye(4)], _placement_box(c, box), _object_points(c))
        if m[0] is None:
            raise ValueError(_unplaced(c, status[0]))
        m[0]["base"] = None
        return m[0]
    if base is None:
        info = _lib.PlacementInfo()
        drop, contacts, support = (torch.empty(c["dim"] ** 2, dtype=t, device=occ.device) for t in (torch.int32, torch.int32, torch.int16))
        _placement_library("dmnerf_placement_map", occ, _lib.ptr(occ), _lib.ptr(labels, torch.int16), c["dim"], c["level"],
                           _lib.doubles(c["T"], 16), _lib.doubles(c["ext"], 3), C.byref(c["desc"]), _lib.ptr(drop, torch.int32),
                           _lib.ptr(contacts, torch.int32), _lib.ptr(support, torch.int16), C.byref(info))
        return _map_result(c, info, drop, contacts, support, None, None, int(info.points))
    box = _placement_box(c, box)
    m, status = _placement_maps(c, [base], box, _object_points(c))
    if m[0] is None:
        raise ValueError(_unplaced(c, status[0]))
    return m[0]


def _unplaced(c, status):
    """Why dmnerf_placement_maps did not place a base (its status 1 or 2)."""
    if status == 1:
        return "placement: label %d has no solid points after the move" % c["label"]
    return "placement: lift %d takes the moved object's top out of the grid [0, %d]" % (c["lift"], c["dim"] - 1)


def _check_scene(scene, occ, labels):
    """placement's scene: None, or an (occ, labels) pair with the shape, dtypes and device of occ / labels."""
    if scene is None:
        return None
    try:
        s_occ, s_lab = scene
    except (TypeError, ValueError):
        raise ValueError("placement: scene must be an (occ, labels) pair") from None
    if not (torch.is_tensor(s_occ) and torch.is_tensor(s_lab)) or s_occ.shape != occ.shape or s_lab.shape != labels.shape or \
            s_occ.dtype != occ.dtype or s_lab.dtype != labels.dtype or s_occ.device != occ.device or s_lab.device != labels.device:
        raise ValueError("placement: the scene must be (occ, labels) tensors of the grid's shape, dtypes and device")
    return s_occ, s_lab


def _placement_call(occ, labels, scene_transform, label, down, lift, extents, level, piece, rest, obstacles, scene=None, copy=False,
                    group=None):
    """The checked arguments of a placement call: grid, level, label, lift, down axis, scene, copy, group and the ABI placement."""
    from .manipulator import _piece_region, move_pieces, move_rests
    from .mesh import EXTENTS, check_transform
    T = check_transform(scene_transform)
    ext = EXTENTS if extents is None else extents
    label = _labels([label], MAX_LABELS - 1, "placement")[0]
    level = _check_level(level)
    if isinstance(lift, (bool, np.bool_)) or int(lift) != lift or int(lift) < 0:
        raise ValueError("placement: lift must be an integer >= 0 voxels, got %r" % (lift,))
    rest_drop = move_rests(rest, 1)[0]
    copy = _check_copies(copy, [label], [rest_drop])[0]
    sets = move_groups(None if group is None else [group], [label], MAX_LABELS - 1, "placement")
    group = None if sets is None else sets[0]
    words = ALL_LABELS if obstacles is None else label_words(obstacles)
    A, _ = grid_affine(T, 2, ext)
    axis, sign = down_axis((A / np.linalg.norm(A, axis=0)).T, down, "placement")
    dim = _check_sweep(occ, labels, "placement_map")
    scene = _check_scene(scene, occ, labels)
    if (copy or group is not None) and scene is None:  # a copy's source stands in the grid it is sampled from
        scene = (occ, labels)
    if not 2 <= dim <= PLACE_MAX_DIM:
        raise ValueError("placement: dim %d outside [2, %d]" % (dim, PLACE_MAX_DIM))
    if int(lift) > dim - 1:
        raise ValueError("placement: lift %d takes the object out of the grid [0, %d]" % (int(lift), dim - 1))
    move_pieces(None if piece is None else [piece], [label], MAX_LABELS - 1, occ.device)
    desc = _lib.Placement(piece=_piece_region(piece, label, MAX_LABELS - 1, occ.device), label=label, rest_drop=int(rest_drop),
                          axis=axis, sign=sign, lift=int(lift))
    desc.obstacles[:] = words
    return {"occ": occ, "labels": labels, "T": T, "ext": ext, "level": level, "label": label, "lift": int(lift), "axis": axis,
            "sign": sign, "dim": dim, "desc": desc, "piece": piece, "scene": scene, "copy": copy, "group": group}


def _placement_library(name, occ, *args):
    try:
        get_context(occ.device).call(name, get_context(occ.device).handle, *args)
    except RuntimeError as e:
        if "(status 1)" in str(e):                     # the library rejected the input: a label without points, the lift, the grid
            raise ValueError(str(e)) from None
        raise


def _placement_box(c, box):
    """The source box of a moved placement: edit_boxes' (margin 2) unless one is given -> int [6]."""
    if box is not None:
        return box
    return edit_boxes(c["occ"], c["labels"], [(c["label"], np.eye(4))], c["T"], c["ext"], c["level"], 2,
                      None if c["piece"] is None else [c["piece"]], None if c.get("group") is None else [c["group"]])[0]


def _object_mask(c):
    if c.get("group") is not None:
        return _group_mask(c["occ"], c["labels"], c["group"], c["level"], c["piece"], c["T"], c["ext"])
    mask = (c["labels"] == c["label"]) & (c["occ"] > c["level"])
    if c["piece"] is not None:
        mask &= _region_keeps(c["piece"], c["T"], c["dim"], c["ext"], c["occ"].device)
    return mask


def _object_points(c):
    return int(_object_mask(c).sum())


def _map_result(c, info, drop, contacts, support, base, box, points_before):
    U, V = int(info.offsets[0]), int(info.offsets[1])
    axis, sign, dim = c["axis"], c["sign"], c["dim"]
    horizontal = [a for a in range(3) if a != axis]
    n = int(info.points)
    centre = [None] * 3
    for a, s in zip(horizontal, info.sum[:2]):
        centre[a] = Fraction(int(s), n)
    ysum = Fraction(int(info.sum[2]), n)                 # heights y: idx_axis, or dim - 1 - idx_axis when +e_axis points down
    centre[axis] = dim - 1 - ysum if sign > 0 else ysum
    return {"drop": drop[:U * V].view(U, V), "support": support[:U * V].view(U, V), "contacts": contacts[:U * V].view(U, V),
            "offset_lo": (int(info.offset_lo[0]), int(info.offset_lo[1])), "axis": axis, "sign": sign, "horizontal": horizontal,
            "centre": centre, "runs": int(info.runs), "points": n, "height": (int(info.height[0]), int(info.height[1])),
            "lift": c["lift"], "label": c["label"], "dim": dim, "base": base, "box": None if box is None else tuple(int(x) for x in box),
            "points_before": points_before,
            "_call": (c["occ"], c["labels"], c["T"], c["ext"], c["level"], c["desc"], c["piece"]), "_scene": c.get("scene"),
            "copy": bool(c.get("copy")), "group": c.get("group")}


def _placement_maps(c, bases, box, points_before):
    """dmnerf_placement_maps for the checked bases (at most MAX_BASES) -> (one placement_map result per base, None where the
    base leaves no point or its top out of the grid; the statuses)."""
    n, dim = len(bases), c["dim"]
    occ = c["occ"]
    drop, contacts = (torch.empty((n, dim * dim), dtype=torch.int32, device=occ.device) for _ in range(2))
    support = torch.empty((n, dim * dim), dtype=torch.int16, device=occ.device)
    infos = (_lib.PlacementInfo * n)()
    status = np.zeros(n, dtype=np.int32)
    rows = np.ascontiguousarray([np.asarray(b, dtype=np.float64)[:3].reshape(-1) for b in bases])
    grids = (_lib.ptr(occ), _lib.ptr(c["labels"], torch.int16))
    name, copy = "dmnerf_placement_maps", ()
    if c.get("scene") is not None:
        grids += (_lib.ptr(c["scene"][0]), _lib.ptr(c["scene"][1], torch.int16))
        name = "dmnerf_placement_maps_in_scene"
    if c.get("copy"):
        name, copy = "dmnerf_placement_maps_in_scene_copy", (1,)
    if c.get("group") is not None:
        name, copy = "dmnerf_placement_maps_in_scene_group", (int(bool(c.get("copy"))), _group_words([c["group"]]))
    _placement_library(name, occ, *grids, dim, c["level"], _lib.doubles(c["T"], 16), _lib.doubles(c["ext"], 3), C.byref(c["desc"]),
                       *copy, rows.ctypes.data_as(C.POINTER(C.c_double)), (C.c_int32 * 6)(*[int(x) for x in box]), n,
                       _lib.ptr(drop, torch.int32), _lib.ptr(contacts, torch.int32), _lib.ptr(support, torch.int16), infos,
                       status.ctypes.data_as(C.POINTER(C.c_int32)))
    maps = [None if status[i] else _map_result(c, infos[i], drop[i], contacts[i], support[i], np.asarray(bases[i], dtype=np.float64),
                                               box, points_before) for i in range(n)]
    return maps, status.tolist()


def placement_delta(m, u, v, drop):
    """The index displacement [3] (int) of the placement at offset (u, v) with `drop`: (u, v) on the horizontal axes and
    lift - drop in height, along -sign on the down axis."""
    delta = [0, 0, 0]
    delta[m["horizontal"][0]], delta[m["horizontal"][1]] = int(u), int(v)
    delta[m["axis"]] = -m["sign"] * (m["lift"] - int(drop))
    return delta


def placement_transform(A, delta):
    """translate(-A delta) (4x4 float64): the move that lands the object at x + A delta, as move_overlap and edited_sweep read it."""
    return _translate(-(np.asarray(A, dtype=np.float64) @ np.asarray(delta, dtype=np.float64)))


def hull_contains(cells, num, den):
    """Whether the point num / den (num: 2 integers, den: an integer > 0) lies in the closed convex hull of the integer points
    `cells` [n, 2]; exact: integer cross products on the points scaled by den.  False without cells."""
    pts = sorted({(int(a) * den, int(b) * den) for a, b in cells})
    q = (int(num[0]), int(num[1]))
    if not pts:
        return False

    def cross(o, a, b):
        return (a[0] - o[0]) * (b[1] - o[1]) - (a[1] - o[1]) * (b[0] - o[0])
    hull = []
    for part in (pts, pts[::-1]):                      # Andrew's monotone chain, collinear points dropped
        chain = []
        for p in part:
            while len(chain) >= 2 and cross(chain[-2], chain[-1], p) <= 0:
                chain.pop()
            chain.append(p)
        hull += chain[:-1]
    if len(hull) <= 2:                                 # a point or a segment: q on it
        a, b = pts[0], pts[-1]
        return cross(a, b, q) == 0 and min(a[0], b[0]) <= q[0] <= max(a[0], b[0]) and min(a[1], b[1]) <= q[1] <= max(a[1], b[1])
    return all(cross(hull[i], hull[(i + 1) % len(hull)], q) >= 0 for i in range(len(hull)))


def placement(m, u, v):
    """The placement of placement_map's result `m` at offset (u, v) (voxels; ValueError outside the map or where it is blocked):
      transformation: the 4x4 (nested list) that lands the object there, as rigid_rays, manipulate_frame, edited_sweep and
                      move_overlap read it: base @ translate(-A delta) (base = I without one);
      offset, drop, support, supported (support >= 0);
      contacts:       the support cells [(h1, h2, label below), ...] (dmnerf_placement_contacts, or _moved with a base), one per
                      resting run;
      stable:         the object's centre of mass projects into the closed convex hull of the support cells (exact);
      centre:         the placed centre of mass A (c + delta) + b, network frame (c: the object's exact centre as m has it)."""
    u, v = int(u), int(v)
    (u0, v0), (U, V) = m["offset_lo"], tuple(m["drop"].shape)
    if not (u0 <= u < u0 + U and v0 <= v < v0 + V):
        raise ValueError("placement: offset (%d, %d) outside [%d, %d] x [%d, %d]" % (u, v, u0, u0 + U - 1, v0, v0 + V - 1))
    drop = int(m["drop"][u - u0, v - v0])
    if drop < 0:
        raise ValueError("placement: offset (%d, %d) is blocked: the raised object overlaps an obstacle" % (u, v))
    support, n = int(m["support"][u - u0, v - v0]), int(m["contacts"][u - u0, v - v0])
    occ, labels, T, ext, level, desc, _ = m["_call"]
    cells = np.zeros((max(n, 1), 3), dtype=np.int32)
    got, dr = C.c_int64(0), C.c_int32(0)
    ctx = get_context(occ.device)
    head = (ctx.handle, _lib.ptr(occ), _lib.ptr(labels, torch.int16), m["dim"], level, _lib.doubles(T, 16), _lib.doubles(ext, 3),
            C.byref(desc))
    tail = (u, v, cells.ctypes.data_as(C.POINTER(C.c_int32)), n, C.byref(got), C.byref(dr))
    scene = m.get("_scene")
    if scene is not None:                              # the scene of the map: the object from occ / labels (identity base by default)
        base = np.eye(4) if m.get("base") is None else m["base"]
        name, copy = ("dmnerf_placement_contacts_in_scene_copy", (1,)) if m.get("copy") else ("dmnerf_placement_contacts_in_scene", ())
        if m.get("group") is not None:
            name, copy = "dmnerf_placement_contacts_in_scene_group", (int(bool(m.get("copy"))), _group_words([m["group"]]))
        ctx.call(name, ctx.handle, _lib.ptr(occ), _lib.ptr(labels, torch.int16), _lib.ptr(scene[0]), _lib.ptr(scene[1], torch.int16),
                 *head[3:], *copy, _lib.doubles(base[:3], 12), (C.c_int32 * 6)(*m["box"]), *tail)
    elif m.get("base") is None:
        ctx.call("dmnerf_placement_contacts", *head, *tail)
    else:
        ctx.call("dmnerf_placement_contacts_moved", *head, _lib.doubles(m["base"][:3], 12), (C.c_int32 * 6)(*m["box"]), *tail)
    if int(got.value) != n or int(dr.value) != drop:
        raise RuntimeError("placement: the grid changed since placement_map (offset (%d, %d): drop %d, %d resting runs; now %d, %d)"
                           % (u, v, drop, n, int(dr.value), int(got.value)))
    cells = cells[:n]
    h1, h2 = m["horizontal"]
    den = m["points"]
    num = (m["centre"][h1] * den + u * den, m["centre"][h2] * den + v * den)
    delta = placement_delta(m, u, v, drop)
    A, b = grid_affine(T, m["dim"], ext)
    centre = A @ (np.array([float(c) for c in m["centre"]]) + np.asarray(delta, dtype=np.float64)) + b
    trans = placement_transform(A, delta)
    if m.get("base") is not None:
        trans = m["base"] @ trans
    return {"transformation": trans.tolist(), "offset": (u, v), "drop": drop, "support": support,
            "supported": support >= 0, "contacts": [tuple(int(x) for x in c) for c in cells],
            "stable": hull_contains(cells[:, :2], num, den), "centre": centre, "delta": delta}


def _turn_cos_sin(angle):
    """cos and sin of `angle` degrees, exactly 0 and +-1 at multiples of 90 (np.cos(np.pi / 2) is not 0)."""
    q, r = divmod(float(angle), 90.0)
    if r == 0.0:
        return ((1.0, 0.0), (0.0, 1.0), (-1.0, 0.0), (0.0, -1.0))[int(q) % 4]
    t = np.radians(float(angle))
    return float(np.cos(t)), float(np.sin(t))


def turn_bases(scene_transform, dim, axis, centre, box, angles, extents=None):
    """The moves that turn an object about the down index axis (DESIGN.md, "Turned placements"), one per angle (degrees) ->
    [(angle, 4x4 base or None when the turned object does not fit the grid horizontally)].
      axis:   the down index axis; the turn is right-handed about A[:, axis] / |A[:, axis]| (network frame);
      centre: the object's exact centre in index space (3 numbers or Fractions); the pivot is the grid point nearest it;
      box:    the object's solid index box (i_lo, i_hi, j_lo, j_hi, k_lo, k_hi).
    The object turned by theta about the pivot P, then shifted by whole voxels so that the pivot's column is the grid's middle
    column, lands at L(x) = R (x - P) + P + A s; its base is L^-1 = [R^T | P - R^T (P + A s)], as move_overlap reads a move.  A
    turn does not fit when a horizontal corner of the box grown by half a voxel, carried by L, leaves [-0.5, dim - 0.5]."""
    T = np.asarray(scene_transform, dtype=np.float64)
    A, b = grid_affine(T, dim, extents)
    n = A[:, axis] / np.linalg.norm(A[:, axis])
    pivot = np.array([int(np.floor(Fraction(x) + Fraction(1, 2))) for x in centre], dtype=np.float64)
    shift = np.zeros(3)
    for a in range(3):
        if a != axis:
            shift[a] = (dim - 1) // 2 - pivot[a]
    P, Ainv = A @ pivot + b, np.linalg.inv(A)
    box = np.asarray(box, dtype=np.float64)
    corners = np.array([[box[2 * a + ((k >> a) & 1)] + (0.5 if (k >> a) & 1 else -0.5) for a in range(3)] for k in range(8)])
    cross = np.array([[0.0, -n[2], n[1]], [n[2], 0.0, -n[0]], [-n[1], n[0], 0.0]])
    out = []
    for angle in angles:
        c, s = _turn_cos_sin(angle)
        R = c * np.eye(3) + s * cross + (1.0 - c) * np.outer(n, n)
        landed = ((corners @ A.T + b - P) @ R.T + P + A @ shift - b) @ Ainv.T
        h = [a for a in range(3) if a != axis]
        if (landed[:, h] < -0.5 - 1e-9).any() or (landed[:, h] > dim - 0.5 + 1e-9).any():
            out.append((float(angle), None))
            continue
        base = np.eye(4)
        base[:3, :3] = R.T
        base[:3, 3] = P - R.T @ (P + A @ shift)
        out.append((float(angle), base))
    return out


def _turn_angles(turns):
    """place_object's turns -> [degrees]: K (an integer >= 1) gives 360 k / K, k = 0 .. K - 1; else a non-empty list of finite
    numbers."""
    if isinstance(turns, (bool, np.bool_)):
        raise ValueError("placement: turns must be an integer >= 1 or a list of degrees, got %r" % (turns,))
    if isinstance(turns, (int, np.integer)):
        if int(turns) < 1:
            raise ValueError("placement: turns must be an integer >= 1 or a list of degrees, got %r" % (turns,))
        return [360.0 * k / int(turns) for k in range(int(turns))]
    try:
        angles = [float(x) for x in turns]
    except (TypeError, ValueError):
        raise ValueError("placement: turns must be an integer >= 1 or a list of degrees, got %r" % (turns,)) from None
    if not angles or not np.isfinite(angles).all():
        raise ValueError("placement: turns must be an integer >= 1 or a non-empty list of finite degrees, got %r" % (turns,))
    return angles


def place_object(occ, labels, scene_transform, label, down, near, on=None, stable=True, lift=0, max_tests=64, extents=None,
                 level=0.45, piece=None, rest="keep", obstacles=None, turns=None, scene=None, copy=False, group=None):
    """The placement of object `label` (or its piece) closest to the network-frame point `near`: over placement_map's offsets
    that are not blocked and rest on an obstacle whose label is in `on` (default: any), ordered by the distance of the placed
    centre of mass from `near` across the down axis (ties: the lowest (u, v)), the first that is stable -- testing at most
    max_tests of them -- or, with stable=False, the first.  turns (DESIGN.md, "Turned placements"): None places the object as it
    lies; an integer K also turns it about the down axis by 360 k / K degrees, a list by those degrees (turn_bases), every turn
    mapped in batched calls; candidates of all turns are ordered by distance, then turn order, then (u, v).  Returns
    {"placement": placement() of it, or None; "reason": None, or why there is none; "candidates": how many offsets qualified;
    "tested": stability tests run; "map": the placement_map result it came from (without turns: the map); "turn": its angle
    (None without turns); "maps": [(angle, map)] of the turns that were mapped; "unfit": the angles whose turned object does not
    fit the grid; "unplaced": the angles whose turned object has no point or leaves the grid at this lift}.  scene, copy: as
    placement_map's (DESIGN.md, "Arranging objects", "Copying objects"); the placement of a copy is the copy's move.  group: as
    placement_map's (DESIGN.md, "Moving objects together"); `on` may name no label of the group, except for a copy."""
    near = _check_point(near, "near")
    if isinstance(max_tests, (bool, np.bool_)) or int(max_tests) != max_tests or int(max_tests) < 1:
        raise ValueError("placement: max_tests must be an integer >= 1, got %r" % (max_tests,))
    on = None if on is None else set(_labels(on, MAX_LABELS - 1, "placement"))
    if group is not None and on is not None and not copy:
        inside = sorted(on & set(_labels(group, MAX_LABELS - 1, "placement")))
        if inside:
            raise ValueError("placement: on names label(s) %s of the moved group: a group never rests on itself" % inside)
    angles = None if turns is None else _turn_angles(turns)
    if turns is None:
        m = placement_map(occ, labels, scene_transform, label, down, lift, extents, level, piece, rest, obstacles, scene=scene,
                          copy=copy, group=group)
        maps, unfit, unplaced = [(None, m)], [], []
    else:
        maps, unfit, unplaced = turned_placement_maps(occ, labels, scene_transform, label, down, angles, lift, extents, level, piece,
                                                      rest, obstacles, scene, copy, group)
    out = {"placement": None, "reason": None, "candidates": 0, "tested": 0, "map": maps[0][1] if turns is None else None,
           "turn": None, "maps": [] if turns is None else maps, "unfit": unfit, "unplaced": unplaced}
    rows = placement_candidates([m for _, m in maps], near, on)
    if rows.shape[0] == 0:
        out["reason"] = "no offset rests on %s" % ("an obstacle" if on is None else "label(s) %s" % sorted(on))
        if turns is not None and not maps:
            out["reason"] = "no turn fits the grid" if not unplaced else "no turned object can be placed"
        return out
    out["candidates"] = int(rows.shape[0])
    for k in range(min(int(max_tests), rows.shape[0])):
        angle, m = maps[int(rows[k, 1])]
        p = placement(m, int(rows[k, 2]), int(rows[k, 3]))
        out["tested"] += 1
        if p["stable"] or not stable:
            out.update(placement=p, map=m, turn=angle)
            return out
    out["reason"] = "none of the %d nearest of %d resting offsets is stable" % (min(int(max_tests), rows.shape[0]), rows.shape[0])
    return out


def turned_placement_maps(occ, labels, scene_transform, label, down, turns, lift=0, extents=None, level=0.45, piece=None,
                          rest="keep", obstacles=None, scene=None, copy=False, group=None):
    """placement_map of the object turned about the down axis by each of `turns` (degrees, or an integer K: 360 k / K), the
    turns built by turn_bases from the object's solid box and exact centre, mapped in dmnerf_placement_maps calls of at most
    MAX_BASES bases, with edit_boxes' source box -> ([(angle, map)] of the turns mapped, the angles that do not fit the grid,
    the angles whose turned object has no point or its top out of the grid).  scene, copy: as placement_map's; the turns are
    built from the object in occ / labels.  group: as placement_map's; the group turns as one body about its centre."""
    angles = _turn_angles(turns)
    c = _placement_call(occ, labels, scene_transform, label, down, lift, extents, level, piece, rest, obstacles, scene, copy, group)
    points, box, centre = _object_extent(_object_mask(c))
    if points == 0:
        raise ValueError("placement: label %d has no solid points%s" % (c["label"], " in its piece" if piece is not None else ""))
    fitted = turn_bases(c["T"], c["dim"], c["axis"], centre, box, angles, c["ext"])
    unfit = [a for a, bs in fitted if bs is None]
    fitted = [(a, bs) for a, bs in fitted if bs is not None]
    src = _placement_box(c, None)
    maps, unplaced = [], []
    for k in range(0, len(fitted), _lib.MAX_BASES):
        chunk = fitted[k:k + _lib.MAX_BASES]
        got, _ = _placement_maps(c, [bs for _, bs in chunk], src, points)
        maps += [(a, mk) for (a, _), mk in zip(chunk, got) if mk is not None]
        unplaced += [a for (a, _), mk in zip(chunk, got) if mk is None]
    return maps, unfit, unplaced


def placement_candidates(maps, near, on=None):
    """The resting offsets of placement_map results `maps` (one per turn, in turn order) that rest on an obstacle (whose label
    is in `on`, when given), in place_object's order: by the distance of the placed centre of mass from the network-frame point
    `near` across the down axis, then by turn, then by (u, v) -> float [n, 4] rows (distance, turn, u, v)."""
    rows = [np.zeros((0, 4))]
    for t, m in enumerate(maps):
        drop, support = m["drop"].cpu().numpy(), m["support"].cpu().numpy()
        ok = (drop >= 0) & (support >= 0)
        if on is not None:
            ok &= np.isin(support, sorted(on))
        iu, iv = np.nonzero(ok)
        T, ext = m["_call"][2], m["_call"][3]
        A, b = grid_affine(T, m["dim"], ext)
        u, v = iu + m["offset_lo"][0], iv + m["offset_lo"][1]
        cm = np.array([float(x) for x in m["centre"]])
        delta = np.zeros((iu.size, 3))
        delta[:, m["horizontal"][0]], delta[:, m["horizontal"][1]] = u, v
        delta[:, m["axis"]] = -m["sign"] * (m["lift"] - drop[iu, iv])
        gap = (cm[None, :] + delta) @ A.T + b - np.asarray(near, dtype=np.float64)[None, :]
        axis_dir = A[:, m["axis"]] / np.linalg.norm(A[:, m["axis"]])
        gap -= np.outer(gap @ axis_dir, axis_dir)
        rows.append(np.stack([np.linalg.norm(gap, axis=1), np.full(iu.size, t), u, v], 1))
    rows = np.concatenate(rows)
    return rows[np.lexsort((rows[:, 3], rows[:, 2], rows[:, 1], rows[:, 0]))]


def _object_extent(mask):
    """The points, solid index box (i_lo, i_hi, j_lo, j_hi, k_lo, k_hi) and exact centre (3 Fractions) of a bool grid's points."""
    n = int(mask.sum())
    if n == 0:
        return 0, EMPTY_BOX, None
    box, centre = [], []
    for a in range(3):
        per = mask.sum(dim=tuple(x for x in range(3) if x != a)).long()
        idx = torch.nonzero(per).flatten()
        box += [int(idx[0]), int(idx[-1])]
        centre.append(Fraction(int((per * torch.arange(per.numel(), device=per.device)).sum()), n))
    return n, tuple(box), centre


def largest_component_grid(occ, labels, level, objects):
    """int16 grid: label k at the points of the largest 26-connected component of each label k of `objects`, -1 elsewhere."""
    cc = object_components(occ, labels, level, 26)
    best = largest_components(cc["label"], cc["voxels"])
    lut = np.full(cc["label"].shape[0], -1, dtype=np.int16)
    for k in objects:
        if int(k) in best:
            lut[best[int(k)]] = int(k)
    return component_groups(cc["grid"], lut, -1)


# ----------------------------------------------------------------------------------------------------------------- arrangement
# DESIGN.md, "Arranging objects": the edited sweep's rule with the network replaced by the unedited grid at the nearest index
# (edited_grid), and several objects placed one after another, each in the scene the earlier placements leave (arrange_objects).
ARRANGE_KEYS = ("label", "near", "on", "piece", "rest", "turns", "stable", "lift", "obstacles", "copy", "group")


def _grid_edit(src_occ, src_labels, occ, labels, T, ext, level, mv, mats, boxes, drops, regions, flags=None, sets=None, defs=None):
    """dmnerf_grid_edit of checked moves (flags: the checked copy flags, None for none; sets: the checked label sets, None for
    none; defs: the checked deformations, None for none): applied in place to occ / labels, sampled from src_occ / src_labels ->
    edited_grid's report."""
    n, dim = len(mv), occ.shape[0]
    overwritten = np.zeros((n, MAX_LABELS), dtype=np.int64)
    landed = np.zeros(n, dtype=np.int64)
    ctx = get_context(occ.device)
    head = (ctx.handle, _lib.ptr(src_occ), _lib.ptr(src_labels, torch.int16), dim, level, _lib.doubles(T, 16), _lib.doubles(ext, 3),
            _edit_moves(mv, mats, boxes, drops, regions, occ.device))
    tail = (n, _lib.ptr(occ), _lib.ptr(labels, torch.int16), landed.ctypes.data_as(C.POINTER(C.c_int64)),
            overwritten.ctypes.data_as(C.POINTER(C.c_int64)))
    if defs is not None:
        ctx.call("dmnerf_grid_edit_deformed", *head, _copy_flags(flags or [False] * n), None if sets is None else _group_words(sets),
                 _deformation_array(defs), *tail)
    elif sets is not None:
        ctx.call("dmnerf_grid_edit_groups", *head, _copy_flags(flags or [False] * n), _group_words(sets), *tail)
    elif flags is not None and any(flags):
        ctx.call("dmnerf_grid_edit_copies", *head, _copy_flags(flags), *tail)
    else:
        ctx.call("dmnerf_grid_edit", *head, *tail)
    unit = _voxel_volume(T, ext, dim)
    return [_count_report(mv[i], landed[i], overwritten[i], unit, "overwritten") for i in range(n)]


def edited_grid(occ, labels, scene_transform, moves, extents=None, level=0.45, boxes=None, margin=2, pieces=None, rest="keep",
                copies=None, groups=None, deformations=None):
    """dmnerf_grid_edit: edited_sweep's moves applied in order to the labelled keep-all sweep occ / labels ([dim]^3 float32 / int16
    on the device) without the network: a move shows at p the unedited grid at the nearest grid index of trans p, as the collision
    checks sample a moved object.  On a grid whose points and steps are exact in fp32, whole-voxel translations and quarter turns
    give edited_sweep's grid bit for bit; elsewhere it is the sweep resampled at its own resolution.  boxes, margin, pieces, rest:
    as edited_sweep (default boxes: edit_boxes of occ / labels).  Works on copies -> (occ', labels', report), report one dict per
    move: label, landed (the voxels it takes from a solid target), overwritten {label: voxels} (labels with voxels > 0: solid
    points of the grid as the earlier moves left it that it lands on and does not vacate), overwritten_volume and total.
    copies: as edited_sweep (DESIGN.md, "Copying objects"); a copy's overwritten counts its own label's points too.  groups: as
    edited_sweep (DESIGN.md, "Moving objects together"); landed and overwritten count the whole set.  deformations: as
    edited_sweep (DESIGN.md, "Deforming objects")."""
    from .manipulator import move_pieces, move_rests
    from .mesh import EXTENTS, check_transform
    T = check_transform(scene_transform)
    dim = _check_sweep(occ, labels, "edited_grid")
    ext = EXTENTS if extents is None else extents
    mv, mats = _check_moves(moves, MAX_LABELS - 1)
    level = _check_level(level)
    drops = move_rests(rest, len(mv))
    sets = move_groups(groups, mv, MAX_LABELS - 1)
    flags = _check_copies(copies, mv, drops, sets=sets)
    defs = move_deformations(deformations, len(mv))
    regions = move_pieces(pieces, mv, MAX_LABELS - 1, occ.device) or [None] * len(mv)
    if int(margin) != margin or int(margin) < 0:
        raise ValueError("edit: margin must be an integer >= 0, got %r" % (margin,))
    if boxes is None:
        boxes = edit_boxes(occ, labels, moves, T, ext, level, margin, pieces, sets)
    boxes = _check_boxes(boxes, len(mv), dim)
    out_occ, out_labels = occ.clone(memory_format=torch.contiguous_format), labels.clone(memory_format=torch.contiguous_format)
    if not mv:
        return out_occ, out_labels, []
    return out_occ, out_labels, _grid_edit(occ, labels, out_occ, out_labels, T, ext, level, mv, mats, boxes, drops, regions, flags,
                                           sets, defs)


def _check_items(items, dim, device):
    """arrange_objects' items, checked before any device work -> [dict with every key of ARRANGE_KEYS]."""
    from .manipulator import move_pieces, move_rests
    if isinstance(items, dict) or not hasattr(items, "__iter__"):
        raise ValueError("arrange: items must be a list of dicts")
    items = list(items)
    if not 1 <= len(items) <= _lib.MAX_MOVES:
        raise ValueError("arrange: between 1 and %d items are supported (the render and the mesh take at most %d moves), got %d"
                         % (_lib.MAX_MOVES, _lib.MAX_MOVES, len(items)))
    out, seen = [], {}
    for i, it in enumerate(items):
        if not isinstance(it, dict):
            raise ValueError("arrange: item %d must be a dict, got %r" % (i, type(it).__name__))
        unknown = sorted(set(it) - set(ARRANGE_KEYS))
        if unknown:
            raise ValueError("arrange: item %d: unknown keys %s (known: %s)" % (i, unknown, ", ".join(ARRANGE_KEYS)))
        for k in ("label", "near"):
            if k not in it:
                raise ValueError("arrange: item %d needs %r" % (i, k))
        c = {k: it.get(k) for k in ARRANGE_KEYS}
        c["label"] = _labels([c["label"]], MAX_LABELS - 1, "arrange")[0]
        c["copy"] = False if c["copy"] is None else c["copy"]
        if not isinstance(c["copy"], (bool, np.bool_)):
            raise ValueError("arrange: item %d: copy must be True or False, got %r" % (i, c["copy"]))
        c["copy"] = bool(c["copy"])
        sets = move_groups(None if c["group"] is None else [c["group"]], [c["label"]], MAX_LABELS - 1, "arrange")
        c["group"] = None if sets is None else sets[0]
        for k in c["group"] or (c["label"],):
            kinds = seen.setdefault(k, {})
            if not c["copy"] and "move" in kinds:
                raise ValueError("arrange: items %d and %d share label %d (the second move would also vacate the first one's landed "
                                 "points)" % (kinds["move"], i, k))
            if not c["copy"] and "copy" in kinds:
                raise ValueError("arrange: item %d moves label %d after item %d copies it (the move would also vacate the copy)"
                                 % (i, k, kinds["copy"]))
        for k in c["group"] or (c["label"],):
            seen[k].setdefault("copy" if c["copy"] else "move", i)
        c["near"] = _check_point(c["near"], "near")
        if c["on"] is not None:
            c["on"] = _labels(c["on"], MAX_LABELS - 1, "arrange")
            if c["group"] is not None and not c["copy"] and set(c["on"]) & set(c["group"]):
                raise ValueError("arrange: item %d: on names label(s) %s of its group: a group never rests on itself"
                                 % (i, sorted(set(c["on"]) & set(c["group"]))))
        if c["turns"] is not None:
            _turn_angles(c["turns"])
        c["stable"] = True if c["stable"] is None else c["stable"]
        if not isinstance(c["stable"], (bool, np.bool_)):
            raise ValueError("arrange: item %d: stable must be True or False, got %r" % (i, c["stable"]))
        c["lift"] = 0 if c["lift"] is None else c["lift"]
        if isinstance(c["lift"], (bool, np.bool_)) or int(c["lift"]) != c["lift"] or not 0 <= int(c["lift"]) <= dim - 1:
            raise ValueError("arrange: item %d: lift must be an integer in [0, %d] voxels, got %r" % (i, dim - 1, c["lift"]))
        c["lift"] = int(c["lift"])
        c["rest"] = "keep" if c["rest"] is None else c["rest"]
        if move_rests(c["rest"], 1)[0] and c["copy"]:
            raise ValueError("arrange: item %d: a copy cannot drop the rest of its label (rest 'drop'): it vacates nothing" % i)
        if c["piece"] is not None:
            move_pieces([c["piece"]], [c["label"]], MAX_LABELS - 1, device)
        if c["obstacles"] is not None:
            label_words(c["obstacles"])
        out.append(c)
    return out


def arrange_objects(occ, labels, scene_transform, items, down, extents=None, level=0.45, max_tests=64):
    """Several objects placed one after another (DESIGN.md, "Arranging objects"), greedily in the order given, each in the scene
    the earlier placements leave: the state starts as a copy of the labelled keep-all sweep occ / labels; item k is placed by
    place_object with the object from the unedited grid and scene = the state, and when it is placed its move is applied to the
    state by the grid-only edit (edited_grid's rule, the default box); an item that is not placed stays where it is and is an
    obstacle for the items after it.  items: dicts with label and near (network frame) and optionally on (labels to rest on; an
    earlier item keeps its label where it landed), piece, rest, turns, stable, lift and obstacles, as place_object takes them, and
    copy (DESIGN.md, "Copying objects"; default False): place a copy of the object from the unedited grid, its source standing as
    an obstacle (`on` may name its own label, to stack it on its source).  At most MAX_MOVES items; no two moves of one label, no
    move of a label after a copy of it; copies of one label may repeat and may follow its move.  group (DESIGN.md, "Moving
    objects together"; labels holding the item's label): the item moves its whole set as one body, as placement_map's group; two
    move items whose sets intersect are rejected as two moves of one label.  down: shared by every item.
    Every item is checked before any device work.
    Returns a dict:
      items:  per item, place_object's result and its label; placement None and a reason when it was not placed (its maps were
              computed on the state before its own move and refer to the state's tensors, which later items edit);
      moves:  [(label, 4x4 nested list)] of the placed items in order, and pieces / rest / copies / groups aligned with them:
              manipulate_frame, manipulator_eval, edited_sweep and edited_mesh take them unchanged (copies: edited_sweep,
              edited_mesh, edited_grid and render_moves; groups, a label tuple or None per move: edited_grid, edited_sweep,
              edited_mesh and render_moves);
      occ, labels: the arranged grid, equal to edited_grid(occ, labels, ..., moves, pieces=pieces, rest=rest, copies=copies) bit
              for bit;
      report: edited_grid's report of each placed move (overwritten: what it landed on in the scene left before it)."""
    from .manipulator import move_rests
    from .mesh import EXTENTS, check_transform
    T = check_transform(scene_transform)
    ext = EXTENTS if extents is None else extents
    if not torch.is_tensor(occ) or occ.dim() != 3:
        raise ValueError("arrange: occ must be a [dim, dim, dim] tensor")
    checked = _check_items(items, occ.shape[0], occ.device)
    level = _check_level(level)
    if isinstance(max_tests, (bool, np.bool_)) or int(max_tests) != max_tests or int(max_tests) < 1:
        raise ValueError("placement: max_tests must be an integer >= 1, got %r" % (max_tests,))
    A, _ = grid_affine(T, 2, ext)
    down_axis((A / np.linalg.norm(A, axis=0)).T, down, "arrange")
    dim = _check_sweep(occ, labels, "arrange_objects")
    if not 2 <= dim <= PLACE_MAX_DIM:
        raise ValueError("placement: dim %d outside [2, %d]" % (dim, PLACE_MAX_DIM))
    state_occ, state_labels = occ.clone(memory_format=torch.contiguous_format), labels.clone(memory_format=torch.contiguous_format)
    out = {"items": [], "moves": [], "pieces": [], "rest": [], "copies": [], "groups": [], "occ": state_occ, "labels": state_labels,
           "report": []}
    for it in checked:
        try:
            r = place_object(occ, labels, T, it["label"], down, it["near"], it["on"], it["stable"], it["lift"], max_tests, ext, level,
                             it["piece"], it["rest"], it["obstacles"], it["turns"], scene=(state_occ, state_labels), copy=it["copy"],
                             group=it["group"])
        except ValueError as e:        # found on the device: no solid points (in its piece), or the lift takes its top out
            r = {"placement": None, "reason": str(e)}
        out["items"].append(dict(r, label=it["label"]))
        if r["placement"] is None:
            continue
        trans = r["placement"]["transformation"]
        move = (it["label"], trans)
        pieces = None if it["piece"] is None else [it["piece"]]
        sets = None if it["group"] is None else [it["group"]]
        box = edit_boxes(occ, labels, [move], T, ext, level, 2, pieces, sets)
        out["report"] += _grid_edit(occ, labels, state_occ, state_labels, T, ext, level, [it["label"]],
                                    [np.asarray(trans, dtype=np.float64)], box, move_rests(it["rest"], 1), [it["piece"]], [it["copy"]],
                                    sets)
        out["moves"].append(move)
        out["pieces"].append(it["piece"])
        out["rest"].append(it["rest"])
        out["copies"].append(it["copy"])
        out["groups"].append(it["group"])
    return out


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


# ----------------------------------------------------------------------------------------------------------------- grid views
# DESIGN.md, "Viewing the labelled grid": camera rays cast through a labelled keep-all grid to the first solid, kept voxel, with no
# network: the look of "place, look, adjust" at the cost of one voxel walk per pixel, and the label or piece under a pixel.
def _cast_words(keep, remove):
    """keep= / remove= of the cast (labels in [0, 127]) -> the 4 keep words, or None for every label."""
    if keep is not None and remove is not None:
        raise ValueError("cast_grid: give at most one of keep= or remove=")
    if keep is None and remove is None:
        return None
    words = label_words(_labels(keep if keep is not None else remove, MAX_LABELS - 1, "cast_grid"))
    return words if keep is not None else [~w & 0xFFFFFFFF for w in words]


def _check_rays(rays_o, rays_d, device):
    _lib.need_cuda("cast_grid", rays_o, rays_d)
    if rays_o.shape != rays_d.shape or rays_o.dim() < 1 or rays_o.shape[-1] != 3:
        raise ValueError("cast_grid: rays_o and rays_d must have one shape [..., 3], got %s and %s"
                         % (tuple(rays_o.shape), tuple(rays_d.shape)))
    if rays_o.device != device or rays_d.device != device:
        raise ValueError("cast_grid: the rays must be on the grid's device")
    if rays_o.dtype != torch.float32 or rays_d.dtype != torch.float32:
        raise ValueError("cast_grid: rays must be float32")


def _check_range(near, far, level):
    near, far, level = float(near), float(far), float(level)
    if not (np.isfinite(near) and np.isfinite(far) and near <= far):
        raise ValueError("cast_grid: near %r and far %r must be finite with near <= far" % (near, far))
    if not np.isfinite(level):
        raise ValueError("cast_grid: level %r is not finite" % (level,))
    return near, far, level


def cast_grid(occ, labels, scene_transform, rays_o, rays_d, near, far, extents=None, level=0.45, keep=None, remove=None,
              components=None, normals=True):
    """dmnerf_grid_cast: each ray o + t d (rays_o, rays_d [..., 3] float32 on the grid's device, network frame) cast over
    t in [near, far] through the labelled grid occ / labels ([dim]^3 float32 / int16: occupancy_objects' keep-all sweep, or
    edited_grid's, arrange_objects' or edited_sweep's output) to its first solid voxel (occ > level) whose label is kept (keep= or
    remove=: labels in [0, 127]; default every label).  Grid point q owns the cube [q - 1/2, q + 1/2]^3, so depth is where the
    ray enters that cube, in the units of rays_d as given.  Returns device tensors of the rays' leading shape: depth (float32,
    +inf without a hit), label (int16, -1), voxel (int64 [..., 3] index (i, j, k), -1), point (o + depth d in float32, NaN
    without a hit), normal (float32 [..., 3], 0 without a hit; None when normals=False) and hit (bool).  With components (an
    object_components result of this grid), also piece: the component id at the hit voxel (-1 without a hit).  The picking
    primitive: the label and piece under a pixel come from the ray of that pixel (get_rays_at).  On edited_grid's or
    arrange_objects' grid, grid_view(moves=, source=) traces each hit voxel to the move that placed it and colours it from the
    network at that move's source."""
    from .mesh import EXTENTS, check_transform
    T = check_transform(scene_transform)
    ext = np.asarray(EXTENTS if extents is None else extents, dtype=np.float64).reshape(-1)
    if ext.shape != (3,) or not (np.isfinite(ext).all() and (ext > 0).all()):
        raise ValueError("cast_grid: extents must be 3 finite values > 0")
    near, far, level = _check_range(near, far, level)
    words = _cast_words(keep, remove)
    if components is not None and (not isinstance(components, dict) or "grid" not in components
                                   or tuple(components["grid"].shape) != tuple(occ.shape)):
        raise ValueError("cast_grid: components must be an object_components result of this grid")
    dim = _check_sweep(occ, labels, "cast_grid")
    _check_rays(rays_o, rays_d, occ.device)
    shape = tuple(rays_o.shape[:-1])
    o = rays_o.reshape(-1, 3).contiguous()
    d = rays_d.reshape(-1, 3).contiguous()
    n, dev = o.shape[0], occ.device
    depth = torch.empty(n, dtype=torch.float32, device=dev)
    label = torch.empty(n, dtype=torch.int16, device=dev)
    voxel = torch.empty(n, dtype=torch.int32, device=dev)
    normal = torch.empty((n, 3), dtype=torch.float32, device=dev) if normals else None
    ctx = get_context(dev)
    ctx.call("dmnerf_grid_cast", ctx.handle, _lib.ptr(occ), _lib.ptr(labels, torch.int16), dim, level, _lib.doubles(T, 16),
             _lib.doubles(ext, 3), None if words is None else _lib.keep_mask(words), _lib.ptr(o), _lib.ptr(d), n, near, far,
             _lib.ptr(depth), _lib.ptr(label, torch.int16), _lib.ptr(voxel, torch.int32), _lib.ptr(normal))
    hit = voxel >= 0
    v = voxel.to(torch.int64)
    ijk = torch.where(hit[:, None], torch.stack([v // (dim * dim), (v // dim) % dim, v % dim], -1), torch.full_like(v[:, None], -1))
    point = torch.where(hit[:, None], o + depth[:, None] * d, torch.full_like(o, float("nan")))
    out = {"depth": depth.reshape(shape), "label": label.reshape(shape), "voxel": ijk.reshape(shape + (3,)),
           "point": point.reshape(shape + (3,)), "normal": None if normal is None else normal.reshape(shape + (3,)),
           "hit": hit.reshape(shape)}
    if components is not None:
        grid = components["grid"].reshape(-1)
        out["piece"] = torch.where(hit, grid[v.clamp(min=0)], torch.full_like(voxel, -1)).reshape(shape)
    return out


def _overlaps(a, b):
    """Whether the storage of tensors a and b overlaps."""
    x, y = _lib.ptr(a, a.dtype, strided=True).value, _lib.ptr(b, b.dtype, strided=True).value
    return a.device == b.device and x < y + b.numel() * b.element_size() and y < x + a.numel() * a.element_size()


def _check_edit_view(occ, labels, scene_transform, extents, level, moves, source):
    """grid_view's moves= and source=, checked against the viewed grid before any device work -> True when given."""
    from .mesh import EXTENTS, check_transform
    if moves is None and source is None:
        return False
    if moves is None or source is None:
        raise ValueError("grid_view: moves= and source= come together (the edit and the unedited sweep it was applied to)")
    if not isinstance(moves, MovedScene):
        raise ValueError("grid_view: moves must be an objects.render_moves(...) result, got %r" % (type(moves).__name__,))
    if not isinstance(source, (tuple, list)) or len(source) != 2 or not all(torch.is_tensor(s) for s in source):
        raise ValueError("grid_view: source must be the pair (occ, labels) of the unedited keep-all sweep")
    s_occ, s_lab = source
    if not (torch.is_tensor(occ) and torch.is_tensor(labels)):
        raise ValueError("grid_view: occ and labels must be tensors")
    if tuple(s_occ.shape) != tuple(occ.shape) or tuple(s_lab.shape) != tuple(occ.shape):
        raise ValueError("grid_view: the source grid %s / %s is not the viewed grid's %s" % (tuple(s_occ.shape), tuple(s_lab.shape),
                                                                                            tuple(occ.shape)))
    if s_occ.dtype != torch.float32 or s_lab.dtype != torch.int16:
        raise ValueError("grid_view: the source's occ must be float32 and its labels int16")
    if s_occ.device != occ.device or s_lab.device != occ.device:
        raise ValueError("grid_view: the source is on %s / %s, the viewed grid on %s" % (s_occ.device, s_lab.device, occ.device))
    if moves.device != occ.device:
        raise ValueError("grid_view: the moves were built on %s, the viewed grid is on %s" % (moves.device, occ.device))
    d = moves.abi()
    if occ.dim() != 3 or d.dim != occ.shape[0]:
        raise ValueError("grid_view: the moves index a grid of dim %d, the viewed grid is %s" % (d.dim, tuple(occ.shape)))
    T = check_transform(scene_transform)
    ext = np.asarray(EXTENTS if extents is None else extents, dtype=np.float64).reshape(-1)
    if not np.array_equal(np.asarray(d.transform[:], dtype=np.float64), T.reshape(-1)) or not (
            ext.shape == (3,) and np.array_equal(np.asarray(d.extents[:], dtype=np.float64), ext)):
        raise ValueError("grid_view: the moves were built on another grid (scene_transform or extents differ)")
    if np.float32(d.level) != np.float32(level):
        raise ValueError("grid_view: the moves were built at level %r, the view is at level %r" % (float(d.level), float(level)))
    return True


def _edit_view(occ, labels, moves, source, o, d, c):
    """dmnerf_grid_edit_source on the cast c of the rays (o, d) [..., 3] -> (move int16, colour point, colour direction not
    normalised) of the rays' shape; ValueError when a hit is not where the grid-only edit of source by moves put it."""
    dim = occ.shape[0]
    s_occ, s_lab = (t.contiguous() for t in source)
    if any(_overlaps(s, g) for s in (s_occ, s_lab) for g in (occ, labels)):   # the same grid viewed as its own edit
        s_occ, s_lab = s_occ.clone(), s_lab.clone()
    shape = tuple(o.shape[:-1])
    hit = c["hit"].reshape(-1)
    v = c["voxel"].reshape(-1, 3)
    lin = torch.where(hit, (v[:, 0] * dim + v[:, 1]) * dim + v[:, 2], torch.full_like(v[:, 0], -1)).to(torch.int32)
    of, df = o.reshape(-1, 3).contiguous(), d.reshape(-1, 3).contiguous()
    depth = c["depth"].reshape(-1).contiguous()
    n = of.shape[0]
    move = torch.empty(n, dtype=torch.int32, device=occ.device)
    point = torch.empty((n, 3), dtype=torch.float32, device=occ.device)
    vdir = torch.empty((n, 3), dtype=torch.float32, device=occ.device)
    mismatched = C.c_int64(0)
    ctx = get_context(occ.device)
    ctx.call("dmnerf_grid_edit_source", ctx.handle, _lib.ptr(occ), _lib.ptr(labels, torch.int16), _lib.ptr(s_occ),
             _lib.ptr(s_lab, torch.int16), C.byref(moves.abi()), moves.copy_flags(), moves.group_words(),
             moves.deformation_array(), _lib.ptr(of), _lib.ptr(df), _lib.ptr(depth), _lib.ptr(lin, torch.int32), n,
             _lib.ptr(move, torch.int32), _lib.ptr(point), _lib.ptr(vdir), C.byref(mismatched))
    if mismatched.value:
        raise ValueError("grid_view: %d of %d hit voxels differ from the grid-only edit of source by moves (the viewed grid is not "
                         "edited_grid(source, moves) there); render it with render_moves and render_frame(moves=)"
                         % (mismatched.value, int(hit.sum())))
    return move.to(torch.int16).reshape(shape), point.reshape(shape + (3,)), vdir.reshape(shape + (3,))


def grid_view(occ, labels, scene_transform, H, W, K, c2w, near, far, extents=None, level=0.45, keep=None, remove=None, lut=None,
              model_fine=None, moves=None, source=None):
    """The labelled grid seen from one camera (c2w [4, 4] or [3, 4]) or several (c2w [V, 4, 4]), all views in one cast_grid
    launch.  Pixel (row, col) casts get_rays_k's ray, the ray render_frame renders there.  Returns device maps [V?, H, W] of depth,
    label and hit, and normal [V?, H, W, 3].  With lut (uint8 [L, 3], e.g. tester.pred_label_lut), also image [V?, H, W, 3] uint8:
    tester.colorize's label colours shaded by |n . d/|d||, black where nothing is hit.  With model_fine, also rgb [V?, H, W, 3]
    float32: sigmoid of the first three outputs of mlp_forward_points(model_fine, point, d/|d|) at the hit pixels (0 elsewhere),
    one network query per pixel.  Without moves that colour is meaningful only on an unedited grid: on an edited grid the hit
    points of a moved, copied or deformed object are not where the network holds its colour.
    moves (a render_moves result, the value render_frame(moves=) takes) and source (the pair (occ, labels) of the unedited keep-all
    sweep the moves were built on) come together, for occ / labels = edited_grid(source, moves) or arrange_objects' grid (DESIGN.md,
    "Colouring an edited view").  Each hit voxel is traced through the moves (dmnerf_grid_edit_source): the result gains move
    [V?, H, W] int16, the last move that placed the hit voxel (-1 off hits and where no move did), and with model_fine the colour of
    a moved pixel is the network's at the hit point pulled back through that move, seen along the moved render's direction, as
    render_frame(moves=) samples it; other pixels keep the colour above bit for bit.  The replay must reproduce occ / labels at
    every hit voxel (the check covers the hits only): otherwise ValueError, with the number of differing hits, before the network
    runs -- an edited_sweep grid, for one, holds the network's occupancies and is previewed with render_moves."""
    from .helpers import get_rays_k
    _check_range(near, far, level)
    if int(H) != H or int(W) != W or int(H) < 1 or int(W) < 1:
        raise ValueError("grid_view: H and W must be integers >= 1, got %r x %r" % (H, W))
    H, W = int(H), int(W)
    pose = torch.as_tensor(c2w, dtype=torch.float32)
    single = pose.dim() == 2
    poses = pose[None] if single else pose
    if poses.dim() != 3 or poses.shape[1] not in (3, 4) or poses.shape[2] != 4 or poses.shape[0] < 1:
        raise ValueError("grid_view: c2w must be [4, 4], [3, 4] or [V, 4, 4], got %s" % (tuple(pose.shape),))
    if lut is not None:
        lut = np.asarray(lut)
        if lut.dtype != np.uint8 or lut.ndim != 2 or lut.shape[1] != 3 or lut.shape[0] < 1:
            raise ValueError("grid_view: lut must be uint8 [L, 3]")
    edited = _check_edit_view(occ, labels, scene_transform, extents, level, moves, source)
    _check_sweep(occ, labels, "grid_view")
    if edited:
        _check_sweep(source[0], source[1], "grid_view")
    poses = poses.to(occ.device)
    rays = [get_rays_k(H, W, K, poses[v]) for v in range(poses.shape[0])]
    o = torch.stack([r[0] for r in rays])
    d = torch.stack([r[1] for r in rays])
    c = cast_grid(occ, labels, scene_transform, o, d, near, far, extents, level, keep, remove)
    out = {k: c[k] for k in ("depth", "label", "normal", "hit")}
    if edited:
        out["move"], e_point, e_dir = _edit_view(occ, labels, moves, source, o, d, c)
    if lut is not None or model_fine is not None:
        dirs = d / torch.norm(d, dim=-1, keepdim=True)
    if lut is not None:
        from .tester import colorize
        shade = (c["normal"] * dirs).sum(-1).abs()
        out["image"] = torch.round(colorize(c["label"], lut).float() * shade[..., None]).clamp(0, 255).to(torch.uint8)
    if model_fine is not None:
        from .autograd import mlp_forward_points
        rgb = torch.zeros(o.shape, dtype=torch.float32, device=occ.device)
        hit = c["hit"]
        pts, vd = c["point"], dirs
        if edited:                             # moved pixels: the pulled-back point and direction; the others as without moves
            moved = (out["move"] >= 0)[..., None]
            pts = torch.where(moved, e_point, pts)
            vd = torch.where(moved, e_dir / torch.norm(e_dir, dim=-1, keepdim=True), vd)
        if bool(hit.any()):
            with torch.no_grad():
                rgb[hit] = torch.sigmoid(mlp_forward_points(model_fine, pts[hit], vd[hit])[:, :3])
        out["rgb"] = rgb
    return {k: v[0] for k, v in out.items()} if single else out
