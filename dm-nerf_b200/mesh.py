"""Labelled object meshes on the device: the mesh extraction of the original project (`mesh_main`, tools/mesh_generator.py, with
the helpers of tools/visualizer.py), on the native kernels.

    occupancy sweep -> marching cubes -> scene space -> vertex normals -> small-cluster removal -> label rays -> argmax

`extract_mesh` returns device tensors; `mesh_main` has the original's signature and writes the same two files
(`<expname>.ply`, `color_<expname>.ply`).  Neither needs skimage, trimesh or open3d.  Conventions and the deviations from
skimage / open3d: DESIGN.md, "Mesh extraction"."""
import ctypes as C
import json
import os

import numpy as np
import torch

from . import _lib
from .engine import get_context

EXTENTS = (1.9, 7.0, 7.0)          # mesh_generator.py:26


def _p(t, dtype):
    if t is None:
        return None
    if not t.is_cuda or not t.is_contiguous() or t.dtype != dtype:
        raise RuntimeError("native mesh call needs a contiguous CUDA %s tensor (got %s, %s)" % (dtype, t.dtype, t.device))
    return C.c_void_p(t.data_ptr())


def _f(t):
    return _p(t, torch.float32)


def _i(t):
    return _p(t, torch.int32)


def _doubles(a, n):
    a = np.asarray(a, dtype=np.float64).reshape(-1)
    if a.size != n:
        raise ValueError("expected %d values, got %d" % (n, a.size))
    return (C.c_double * n)(*a.tolist())


def check_transform(scene_transform):
    """The 4x4 scene transform (inv(to_origin) of the scene's oriented bounds) as float64; a reflection is rejected."""
    T = np.asarray(scene_transform, dtype=np.float64)
    if T.shape != (4, 4) or not np.isfinite(T).all():
        raise ValueError("scene_transform must be a finite 4x4 matrix, got shape %s" % (T.shape,))
    if np.linalg.det(T[:3, :3]) <= 0:
        raise ValueError("scene_transform has a non-positive determinant (a reflection or a degenerate matrix): the mesh would "
                         "be turned inside out")
    return T


def grid_points(scene_transform, dim, extents=EXTENTS, begin=0, count=None, device="cuda"):
    """Points [begin, begin + count) of the dim^3 query grid in the network's frame (mesh_generator.py:23-29) -> [count, 3]."""
    T = check_transform(scene_transform)
    count = dim ** 3 - begin if count is None else count
    ctx = get_context(device)
    out = torch.empty((count, 3), device=device, dtype=torch.float32)
    _lib.check(ctx.lib.dmnerf_mesh_grid_points(_doubles(T, 16), _doubles(extents, 3), dim, begin, count, _f(out), ctx.stream()),
               "dmnerf_mesh_grid_points")
    return out


def occupancy_grid(model, scene_transform, grid_dim=256, extents=EXTENTS, near=4.0, far=15.0, N_importance=128, slab=0,
                   device="cuda"):
    """mesh_generator.py:23-63: occupancy 1 - exp(-relu(sigma) * (far - near) / N_importance) of `model` on the grid, with zero
    view directions, evaluated slab by slab (slab <= 0: 2^20 points) -> [grid_dim]^3 on the device."""
    T = check_transform(scene_transform)
    ctx = get_context(device)
    slot = ctx.slot_for(model)
    ctx.bind(slot, model)
    occ = torch.empty((grid_dim,) * 3, device=device, dtype=torch.float32)
    voxel = (far - near) / N_importance
    _lib.check(ctx.lib.dmnerf_mesh_occupancy(ctx.handle, slot, _doubles(T, 16), _doubles(extents, 3), grid_dim, voxel, slab, _f(occ),
                                             ctx.stream()), "dmnerf_mesh_occupancy")
    return occ


def marching_cubes(grid, level=0.45):
    """Marching cubes on a device grid [nx, ny, nz] (inside = value > level) -> verts [V, 3] float32 in index units, tris [T, 3]
    int32 (the role of skimage.measure.marching_cubes(grid, level, gradient_direction='ascent'), mesh_generator.py:68-69).
    A grid holding NaN is rejected."""
    if grid.dim() != 3:
        raise ValueError("marching_cubes: expected a 3-D grid, got shape %s" % (tuple(grid.shape),))
    g = grid.contiguous().float()
    ctx = get_context(g.device)
    nx, ny, nz = g.shape
    counts = (C.c_int64 * 2)()
    _lib.check(ctx.lib.dmnerf_mesh_mc_count(ctx.handle, _f(g), nx, ny, nz, level, counts, ctx.stream()), "dmnerf_mesh_mc_count")
    verts = torch.empty((counts[0], 3), device=g.device, dtype=torch.float32)
    tris = torch.empty((counts[1], 3), device=g.device, dtype=torch.int32)
    _lib.check(ctx.lib.dmnerf_mesh_mc_emit(ctx.handle, _f(g), nx, ny, nz, level, _f(verts), _i(tris), ctx.stream()),
               "dmnerf_mesh_mc_emit")
    return verts, tris


def to_scene(verts, scene_transform, grid_dim, extents=EXTENTS):
    """Index-space vertices -> scene space (mesh_generator.py:70-86)."""
    T = check_transform(scene_transform)
    ctx = get_context(verts.device)
    out = torch.empty_like(verts)
    _lib.check(ctx.lib.dmnerf_mesh_to_scene(_f(verts), verts.shape[0], _doubles(T, 16), _doubles(extents, 3), grid_dim, _f(out),
                                            ctx.stream()), "dmnerf_mesh_to_scene")
    return out


def vertex_normals(verts, tris):
    """Area-weighted unit vertex normals (open3d compute_vertex_normals, visualizer.py:164)."""
    ctx = get_context(verts.device)
    out = torch.empty_like(verts)
    _lib.check(ctx.lib.dmnerf_mesh_normals(ctx.handle, _f(verts), verts.shape[0], _i(tris), tris.shape[0], _f(out), ctx.stream()),
               "dmnerf_mesh_normals")
    return out


def triangle_clusters(tris, n_verts):
    """Edge-connected triangle clusters -> (cluster [T] = smallest triangle index of the cluster, cluster_size [T]), int32."""
    ctx = get_context(tris.device)
    cluster = torch.empty(tris.shape[0], device=tris.device, dtype=torch.int32)
    size = torch.empty_like(cluster)
    _lib.check(ctx.lib.dmnerf_mesh_clusters(ctx.handle, _i(tris), tris.shape[0], n_verts, _i(cluster), _i(size), ctx.stream()),
               "dmnerf_mesh_clusters")
    return cluster, size


def clean_mesh(verts, normals, tris, min_cluster=400):
    """visualizer.clean_mesh(min_num_cluster=min_cluster): triangles of clusters with fewer than min_cluster triangles removed,
    then unreferenced vertices; relative order kept.  Returns (verts, normals, tris)."""
    ctx = get_context(verts.device)
    _, size = triangle_clusters(tris, verts.shape[0])
    ov, on = torch.empty_like(verts), (None if normals is None else torch.empty_like(normals))
    ot = torch.empty_like(tris)
    counts = (C.c_int64 * 2)()
    _lib.check(ctx.lib.dmnerf_mesh_clean(ctx.handle, _f(verts), _f(normals), verts.shape[0], _i(tris), tris.shape[0], _i(size),
                                         int(min_cluster), _f(ov), _f(on), _i(ot), counts, ctx.stream()), "dmnerf_mesh_clean")
    nv, nt = counts[0], counts[1]
    return ov[:nv], (None if on is None else on[:nv]), ot[:nt]


def label_rays(verts, normals, near):
    """Per-vertex label rays in the network's frame (mesh_generator.py:106-113) -> rays_o, rays_d [V, 3]."""
    ctx = get_context(verts.device)
    ro, rd = torch.empty_like(verts), torch.empty_like(verts)
    _lib.check(ctx.lib.dmnerf_mesh_label_rays(_f(verts), _f(normals), verts.shape[0], near, _f(ro), _f(rd), ctx.stream()),
               "dmnerf_mesh_label_rays")
    return ro, rd


def argmax_rows(x):
    """torch.argmax(x, -1) for x [N, C] float32 on the device -> int64 [N]."""
    ctx = get_context(x.device)
    x = x.contiguous()
    out = torch.empty(x.shape[0], device=x.device, dtype=torch.int64)
    _lib.check(ctx.lib.dmnerf_argmax_rows(_f(x), x.shape[0], x.shape[1], C.c_void_p(out.data_ptr()), ctx.stream()),
               "dmnerf_argmax_rows")
    return out


def render_labels(model_coarse, model_fine, rays_o, rays_d, N_samples=64, N_importance=128, N_test=4096):
    """mesh_generator.py:117-136: each ray rendered deterministically with depths z_val_sample(n, 0.01, 15, N_samples), N_test rays
    per call, label = argmax of the fine instance map."""
    from .helpers import z_val_sample
    from .render import render_rays
    z = z_val_sample(1, 0.01, 15, N_samples)[0].to(rays_o.device)
    labels = torch.empty(rays_o.shape[0], device=rays_o.device, dtype=torch.int64)
    for b in range(0, rays_o.shape[0], N_test):
        out = render_rays(rays_o[b:b + N_test], rays_d[b:b + N_test], model_coarse, model_fine, z, N_importance=N_importance,
                          want_raw=False, want_coarse=False)
        labels[b:b + N_test] = argmax_rows(out["ins_fine"])
    return labels


def extract_mesh(model_fine, model_coarse, scene_transform, grid_dim=256, level=0.45, extents=EXTENTS, near=4.0, far=15.0,
                 N_samples=64, N_importance=128, N_test=4096, min_cluster=400):
    """The mesh of mesh_main on the device.  Defaults are the original's (mesh_generator.py:19-26, configs/dmsr/test/meshing.txt).
    Returns device tensors:
      vertices, triangles, normals        the marching-cubes mesh in scene space (written as <expname>.ply) and its normals
      clean_vertices, clean_normals, clean_triangles   after small-cluster removal (written as color_<expname>.ply)
      labels                              int64 object label per clean vertex
      rays_o, rays_d                      the label rays, in the network's frame"""
    T = check_transform(scene_transform)
    dev = next(model_fine.parameters()).device
    with torch.no_grad():
        occ = occupancy_grid(model_fine, T, grid_dim, extents, near, far, N_importance, device=dev)
        v_idx, tris = marching_cubes(occ, level)
        del occ
        verts = to_scene(v_idx, T, grid_dim, extents)
        normals = vertex_normals(verts, tris)
        cv, cn, ct = clean_mesh(verts, normals, tris, min_cluster)
        ro, rd = label_rays(cv, cn, near)
        labels = render_labels(model_coarse, model_fine, ro, rd, N_samples, N_importance, N_test)
    return {"vertices": verts, "triangles": tris, "normals": normals, "clean_vertices": cv, "clean_normals": cn,
            "clean_triangles": ct, "labels": labels, "rays_o": ro, "rays_d": rd}


def label_colors(labels, ins_rgbs, color_dict, ins_map):
    """visualizer.render_label2world on the host: a label found in ins_map gets ins_rgbs[color_dict[str(ins_map[label])]], any other
    label black -> uint8 [N, 3] in ins_rgbs' channel order."""
    labels = np.asarray(labels.cpu() if torch.is_tensor(labels) else labels).reshape(-1)
    rgbs = np.asarray(ins_rgbs)
    out = np.zeros((labels.shape[0], 3))
    for lab in np.unique(labels):
        key = str(int(lab))
        if key in ins_map:
            out[labels == lab] = rgbs[color_dict[str(ins_map[key])]]
    return out.astype(np.uint8)


def write_ply(path, verts, faces, colors=None):
    """Binary little-endian PLY: float32 x y z, optional uchar red green blue per vertex, int32 vertex_indices per face."""
    v = np.ascontiguousarray(np.asarray(verts.cpu() if torch.is_tensor(verts) else verts, dtype=np.float32).reshape(-1, 3))
    f = np.ascontiguousarray(np.asarray(faces.cpu() if torch.is_tensor(faces) else faces, dtype=np.int32).reshape(-1, 3))
    fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    if colors is not None:
        fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
    vrec = np.empty(v.shape[0], dtype=fields)
    vrec["x"], vrec["y"], vrec["z"] = v[:, 0], v[:, 1], v[:, 2]
    if colors is not None:
        c = np.asarray(colors, dtype=np.uint8).reshape(-1, 3)
        if c.shape[0] != v.shape[0]:
            raise ValueError("write_ply: %d colours for %d vertices" % (c.shape[0], v.shape[0]))
        vrec["red"], vrec["green"], vrec["blue"] = c[:, 0], c[:, 1], c[:, 2]
    frec = np.empty(f.shape[0], dtype=[("n", "u1"), ("i", "<i4", (3,))])
    frec["n"], frec["i"] = 3, f
    head = ["ply", "format binary_little_endian 1.0", "element vertex %d" % v.shape[0],
            "property float x", "property float y", "property float z"]
    if colors is not None:
        head += ["property uchar red", "property uchar green", "property uchar blue"]
    head += ["element face %d" % f.shape[0], "property list uchar int vertex_indices", "end_header"]
    with open(path, "wb") as fh:
        fh.write(("\n".join(head) + "\n").encode("ascii"))
        fh.write(vrec.tobytes())
        fh.write(frec.tobytes())


def read_ply(path):
    """Reader of the files write_ply writes -> {"vertices", "faces", "colors" (or None)}."""
    with open(path, "rb") as fh:
        data = fh.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode("ascii").split("\n")
    if "format binary_little_endian 1.0" not in head:
        raise ValueError("read_ply: only binary little-endian PLY is read")
    nv = nf = 0
    props = []
    for line in head:
        w = line.split()
        if w[:2] == ["element", "vertex"]:
            nv = int(w[2])
        elif w[:2] == ["element", "face"]:
            nf = int(w[2])
        elif w[:1] == ["property"] and w[1] != "list":
            props.append((w[2], {"float": "<f4", "uchar": "u1"}[w[1]]))
    vrec = np.frombuffer(data, dtype=props, count=nv, offset=end)
    frec = np.frombuffer(data, dtype=[("n", "u1"), ("i", "<i4", (3,))], count=nf, offset=end + vrec.nbytes)
    if nf and not (frec["n"] == 3).all():
        raise ValueError("read_ply: only triangle faces are read")
    colors = np.stack([vrec["red"], vrec["green"], vrec["blue"]], -1) if "red" in vrec.dtype.names else None
    return {"vertices": np.stack([vrec["x"], vrec["y"], vrec["z"]], -1), "faces": frec["i"].copy(), "colors": colors}


def mesh_main(position_embedder, view_embedder, model_coarse, model_fine, args, trimesh_scene, ins_rgbs, save_dir, ins_map=None,
              scene_transform=None, color_dict=None, **extract_kw):
    """tools/mesh_generator.py mesh_main: writes <save_dir>/<args.expname>.ply (the marching-cubes mesh in scene space) and
    <save_dir>/color_<args.expname>.ply (the cleaned mesh, every vertex coloured by its predicted object).
    scene_transform: 4x4; by default inv(trimesh.bounds.oriented_bounds(trimesh_scene)[0]), which needs trimesh.
    color_dict: by default ./data/color_dict.json[dataset][scene] with dataset / scene from args.datadir, as in the original.
    ins_map: predicted label -> ground-truth label (string keys); None maps every label to itself.
    Reads args.near, far, N_samples, N_importance, N_test, expname (and datadir); extract_kw (grid_dim, level, extents,
    min_cluster) go to extract_mesh.  Returns extract_mesh's dict."""
    from .render import _check_embedders
    _check_embedders(position_embedder, view_embedder)
    if scene_transform is None:
        try:
            import trimesh
        except ImportError:
            raise RuntimeError("mesh_main: trimesh is not installed; pass scene_transform= (the 4x4 inverse of the scene's "
                               "oriented-bounds transform)") from None
        to_origin, _ = trimesh.bounds.oriented_bounds(trimesh_scene)
        scene_transform = np.linalg.inv(to_origin)
    if color_dict is None:
        _, _, dataset_name, scene_name = args.datadir.split("/")
        with open(os.path.join(".", "data", "color_dict.json")) as fh:
            color_dict = json.load(fh)[dataset_name][scene_name]
    out = extract_mesh(model_fine, model_coarse, scene_transform, near=args.near, far=args.far, N_samples=args.N_samples,
                       N_importance=args.N_importance, N_test=args.N_test, **extract_kw)
    write_ply(os.path.join(save_dir, args.expname + ".ply"), out["vertices"], out["triangles"])
    labels = out["labels"].cpu().numpy()
    if ins_map is None:
        ins_map = {str(int(k)): int(k) for k in np.unique(labels)}
    colors = label_colors(labels, ins_rgbs, color_dict, ins_map)[:, ::-1]          # mesh_generator.py:139: channels reversed
    write_ply(os.path.join(save_dir, "color_" + args.expname + ".ply"), out["clean_vertices"], out["clean_triangles"], colors)
    return out
