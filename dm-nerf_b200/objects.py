"""Object selection: render or mesh chosen objects of a trained scene (DESIGN.md, "Object selection").

    object_mask(ins_num, keep=None, remove=None)        -> the 4-word mask of kept labels
    render_objects(position_embedder, view_embedder, model_coarse, model_fine, poses, hwk, args, keep=None, remove=None, ...)
                                                        -> isolated / removed views through the frame driver
    object_meshes(model_fine, model_coarse, scene_transform, objects=None, grid_dim=256, level=0.45, ...)
                                                        -> {label: closed mesh of that object}

Every network sample is labelled argmax(sigmoid(instance logits)) over all ins_num + 1 channels, first maximum winning (the
exchanger's rule); a sample whose label is not kept has alpha = 0 in the composite of both passes, so the coarse weights of the
selected scene drive the importance sampling.  The instance map keeps the network's channels: selection does not re-label it."""
import os

import numpy as np
import torch

from . import _lib

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
                   savedir=None, ins_rgbs=None, color_dict=None, impl=_lib.IMPL_AUTO):
    """Render every pose (camera-to-world, [4, 4] or [3, 4]) with the selection, deterministically, through the frame driver.
    Reads args.near, args.far, args.N_samples, args.N_importance.  Returns one dict per pose of device maps: rgb [H, W, 3],
    ins [H, W, ins_num], depth [H, W], acc [H, W].
    savedir: writes {i:03d}.png (RGBA, alpha = acc: an isolated object is a cut-out) and instance_{i:03d}.png (the arg-max label
    of the instance map, coloured as render_test colours it: ins_rgbs[color_dict[label]], channels in cv2's order).  Without
    ins_rgbs / color_dict, label k gets colour k of a fixed seeded palette.  impl: the network, as in render_frame."""
    from .render import _check_embedders, render_frame
    from .tester import colorize, pred_label_lut, write_png
    _check_embedders(position_embedder, view_embedder)
    H, W, K = hwk
    H, W = int(H), int(W)
    dev = next(model_fine.parameters()).device
    ins_num = int(model_fine.ins_linear.weight.shape[0]) - 1
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
                             N_importance=args.N_importance, device=dev, keep_objects=kept, impl=impl)
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
                  far=15.0, N_importance=128, min_cluster=400):
    """One mesh per object: one selected occupancy sweep of model_fine (keeping `objects`) with the label grid, then
    meshes_from_labelled_grid.  objects: labels in [0, ins_num]; default every label present in the grid except the last
    channel (ins_num, "no object").  model_coarse is accepted for symmetry with extract_mesh and not evaluated: the labels come
    from the fine network's per-point logits, not from rendered rays.  Returns {label: mesh dict} of device tensors."""
    from .mesh import check_transform
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
        return meshes_from_labelled_grid(occ, labels, T, objects, level, extents, min_cluster)
