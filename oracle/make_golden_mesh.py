"""Generate tests/golden/mesh_grid.npz: the mesh-extraction query grid of the UNMODIFIED reference
(tools/visualizer.py make_3D_grid / grid_within_bound, then the axis swap and flip of tools/mesh_generator.py:27-29).

tools/visualizer.py imports open3d and matplotlib at the top, which are not installed here, so only the two grid functions are
taken from that file: their definitions are parsed out of it and executed in a namespace holding torch and numpy.

    python oracle/make_golden_mesh.py
"""
import ast
import os

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFERENCE = os.environ.get("DMNERF_REFERENCE_ROOT", "/root/reference")
OUT = os.path.join(ROOT, "tests", "golden")


def reference_grid_functions():
    path = os.path.join(REFERENCE, "tools", "visualizer.py")
    tree = ast.parse(open(path).read(), path)
    keep = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in ("make_3D_grid", "grid_within_bound")]
    assert len(keep) == 2, "grid functions not found in %s" % path
    ns = {"torch": torch, "np": np}
    exec(compile(ast.Module(body=keep, type_ignores=[]), path, "exec"), ns)
    return ns["grid_within_bound"]


def rigid(rx, ry, rz, t):
    cx, sx, cy, sy, cz, sz = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry), np.cos(rz), np.sin(rz)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    T = np.eye(4)
    T[:3, :3] = Rz @ Ry @ Rx
    T[:3, 3] = t
    return T


def main():
    grid_within_bound = reference_grid_functions()
    extents = np.array([1.9, 7.0, 7.0])
    save = {"extents": extents}
    # scene_transform = inv(to_origin) of an oriented bounding box: a rigid transform in float64 (mesh_generator.py:23-25)
    for tag, dim, T in (("a", 12, np.linalg.inv(rigid(0.31, -0.47, 1.13, [0.42, -1.7, 2.3]))),
                        ("b", 7, rigid(-2.2, 0.05, 0.6, [3.1, 0.25, -0.8]))):
        pts, _ = grid_within_bound([-1.0, 1.0], extents, T, grid_dim=dim)
        pts = pts[:, :, [0, 2, 1]]                                       # mesh_generator.py:28-29
        pts[:, :, 1] = pts[:, :, 1] * -1
        save.update({"transform_" + tag: T, "dim_" + tag: dim, "points_" + tag: pts.reshape(-1, 3).numpy()})
        print("grid %s: dim %d, %d points, |p| max %.3f" % (tag, dim, dim ** 3, float(pts.abs().max())))
    np.savez_compressed(os.path.join(OUT, "mesh_grid.npz"), **save)
    print("written", os.path.join(OUT, "mesh_grid.npz"))


if __name__ == "__main__":
    main()
