"""CPU: mesh extraction host logic -- the query-grid arithmetic against the original's grid (golden), the table-free marching
cubes oracle on analytic fields, PLY round trip, label colouring, the drop-in `tools` package."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import marching_cubes as MC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def grid_points_np(T, extents, dim):
    """The fp32 operation order of grid_points_kernel (mesh.cu), restated in numpy."""
    T = np.asarray(T, dtype=np.float64).astype(np.float32)
    step = np.float32(2.0) / np.float32(dim - 1)
    # torch.linspace(-1, 1, dim): one rounding of step * i - 1 (below half) or 1 - step * (dim - 1 - i)
    t = np.array([np.float32(np.float64(step) * i - 1.0) if i < dim // 2 else np.float32(1.0 - np.float64(step) * (dim - 1 - i))
                  for i in range(dim)], dtype=np.float32)
    s = (np.asarray(extents, dtype=np.float64) / 2.0).astype(np.float32)
    I, J, K = np.meshgrid(np.arange(dim), np.arange(dim), np.arange(dim), indexing="ij")
    q = np.stack([t[I] * s[0], t[J] * s[1], t[K] * s[2]], -1).reshape(-1, 3)
    w = [((T[r, 0] * q[:, 0] + T[r, 1] * q[:, 1]) + T[r, 2] * q[:, 2]) + T[r, 3] for r in range(3)]
    return np.stack([w[0], -w[2], w[1]], -1)


def test_grid_arithmetic_matches_the_original_grid_bit_for_bit(golden_dir):
    g = np.load(os.path.join(golden_dir, "mesh_grid.npz"))
    for tag in "ab":
        mine = grid_points_np(g["transform_" + tag], g["extents"], int(g["dim_" + tag]))
        np.testing.assert_array_equal(mine, g["points_" + tag])


def test_scene_transform_with_a_reflection_is_rejected():
    from dmnerf_b200.mesh import check_transform
    T = np.eye(4)
    check_transform(T)
    T[1, 1] = -1.0
    with pytest.raises(ValueError):
        check_transform(T)
    with pytest.raises(ValueError):
        check_transform(np.eye(3))


def _centered(n):
    x = np.arange(n, dtype=np.float64) - (n - 1) / 2.0
    return np.meshgrid(x, x, x, indexing="ij")


def sphere(n, r):
    X, Y, Z = _centered(n)
    return (r - np.sqrt(X * X + Y * Y + Z * Z)).astype(np.float32)


def torus(n, R, r):
    X, Y, Z = _centered(n)
    return (r - np.sqrt((np.sqrt(X * X + Y * Y) - R) ** 2 + Z * Z)).astype(np.float32)


def edge_counts(tris):
    directed = np.concatenate([tris[:, [0, 1]], tris[:, [1, 2]], tris[:, [2, 0]]])
    und = np.sort(directed, 1)
    _, n_und = np.unique(und, axis=0, return_counts=True)
    _, n_dir = np.unique(directed, axis=0, return_counts=True)
    return n_und, n_dir


def euler(verts, tris):
    n_und, _ = edge_counts(tris)
    return len(verts) - len(n_und) + len(tris)


def test_oracle_sphere_is_closed_oriented_and_has_the_right_volume():
    r = 25.3
    v, t, _ = MC.marching_cubes(sphere(64, r), 0.0)
    n_und, n_dir = edge_counts(t)
    assert (n_und == 2).all() and (n_dir == 1).all()
    assert euler(v, t) == 2
    p = v.astype(np.float64) - 31.5
    a, b, c = p[t[:, 0]], p[t[:, 1]], p[t[:, 2]]
    vol = -np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0      # normals point inward (toward larger values)
    assert abs(vol / (4.0 / 3.0 * np.pi * r ** 3) - 1.0) < 0.01
    # face normals point up the analytic gradient (toward the centre)
    fn = np.cross(b - a, c - a)
    centroid = (a + b + c) / 3.0
    big = np.linalg.norm(fn, axis=1) > 1e-6
    assert (np.einsum("ij,ij->i", fn[big], -centroid[big]) > 0).all()


def test_oracle_torus_has_euler_characteristic_zero():
    v, t, _ = MC.marching_cubes(torus(48, 12.0, 5.2), 0.0)
    n_und, n_dir = edge_counts(t)
    assert (n_und == 2).all() and (n_dir == 1).all()
    assert euler(v, t) == 0


def test_oracle_vertex_position_and_numbering():
    g = np.zeros((2, 3, 2), dtype=np.float32)
    g[1, 2, 1] = 1.0
    g[0, 0, 0] = 0.8
    v, t, ids = MC.marching_cubes(g, 0.45)
    assert (np.diff(ids) > 0).all()
    lev = np.float32(0.45)
    # edge (0,0,0) -> (1,0,0): v0 = 0.8 inside, v1 = 0 outside
    k = list(ids).index(0)
    assert v[k, 0] == np.float32(0.0) + (lev - np.float32(0.8)) / (np.float32(0.0) - np.float32(0.8))
    assert len(t) > 0 and t.max() < len(v)


def test_oracle_ambiguous_faces_keep_inside_corners_apart():
    # two diagonal inside corners of one face, nothing else inside: two separate triangles, not a bridge
    ins = [0] * 8
    ins[0] = ins[3] = 1                                  # corners (0,0,0) and (1,1,0) on the face z = 0
    loops = MC.cell_polygons(ins)
    assert sorted(len(l) for l in loops) == [3, 3]
    # the complement: now the face's inside corners are (1,0,0) and (0,1,0); kept apart, they leave the two outside corners
    # joined across the face, and the surface is one hexagon around that outside tube
    loops = MC.cell_polygons([1 - x for x in ins])
    assert sorted(len(l) for l in loops) == [6]


def test_ply_round_trip(tmp_path):
    from dmnerf_b200.mesh import write_ply, read_ply
    rng = np.random.default_rng(3)
    v = rng.standard_normal((57, 3)).astype(np.float32)
    f = rng.integers(0, 57, (91, 3)).astype(np.int32)
    c = rng.integers(0, 256, (57, 3)).astype(np.uint8)
    write_ply(tmp_path / "a.ply", v, f, c)
    write_ply(tmp_path / "b.ply", torch.from_numpy(v), torch.from_numpy(f))
    a, b = read_ply(tmp_path / "a.ply"), read_ply(tmp_path / "b.ply")
    np.testing.assert_array_equal(a["vertices"], v)
    np.testing.assert_array_equal(a["faces"], f)
    np.testing.assert_array_equal(a["colors"], c)
    np.testing.assert_array_equal(b["vertices"], v)
    assert b["colors"] is None
    head = open(tmp_path / "a.ply", "rb").read(200)
    assert head.startswith(b"ply\nformat binary_little_endian 1.0\nelement vertex 57\n")


def render_label2world(predicted_labels, rgbs, color_dict, ins_map):
    """Restatement of the original's visualizer.render_label2world (tools/visualizer.py:208-223)."""
    unique_labels = torch.unique(predicted_labels)
    out = np.zeros(shape=(predicted_labels.shape[0], 3))
    for label in unique_labels:
        key = str(int(label))
        if key in ins_map.keys():
            out[predicted_labels == label] = rgbs[color_dict[str(ins_map[key])]]
    return out.astype(np.uint8)


def test_label_colours_match_render_label2world():
    from dmnerf_b200.mesh import label_colors
    rng = np.random.default_rng(5)
    rgbs = rng.integers(0, 256, (20, 3))
    color_dict = {str(k): (k * 7) % 20 for k in range(20)}
    ins_map = {"0": 3, "2": 11, "5": 5, "7": 0}
    labels = torch.from_numpy(rng.integers(0, 9, 400))
    np.testing.assert_array_equal(label_colors(labels, rgbs, color_dict, ins_map),
                                  render_label2world(labels, rgbs, color_dict, ins_map))


def test_dropin_tools_package_serves_the_native_mesh_main(tmp_path):
    """`from tools.mesh_generator import mesh_main` resolves to the native function; the original's other tools modules are found
    through the package __path__ (stand-in tree, resolved like the original's)."""
    (tmp_path / "tools").mkdir()
    (tmp_path / "tools" / "visualizer.py").write_text("def clean_mesh(*a, **k): return 'standin'\n")
    (tmp_path / "tools" / "pose_generator.py").write_text("def generate_poses(*a, **k): return 'poses'\n")
    (tmp_path / "tools" / "mesh_generator.py").write_text("def mesh_main(*a, **k): raise AssertionError('stand-in mesh_main')\n")
    env = dict(os.environ, DMNERF_REFERENCE_ROOT=str(tmp_path),
               PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "dm-nerf_b200", "dropin"), ROOT]))
    code = r"""
import dmnerf_b200.mesh as nm
from tools.mesh_generator import mesh_main
assert mesh_main is nm.mesh_main
import tools.visualizer as V, tools.pose_generator as P
assert V.clean_mesh() == "standin" and P.generate_poses() == "poses"
print("ok")
"""
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-3000:]


def test_oracle_noise_field_has_no_face_chords():
    """Fan chords never lie in a cell face: on a field that hits every case, no directed edge repeats and no edge has three
    triangles."""
    g = np.random.default_rng(11).random((24, 21, 19)).astype(np.float32)
    _, t, _ = MC.marching_cubes(g, 0.45)
    n_und, n_dir = edge_counts(t)
    assert (n_dir == 1).all() and n_und.max() == 2
