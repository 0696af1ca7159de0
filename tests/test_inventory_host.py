"""CPU: the object inventory's definitions -- the oracle (oracle/inventory_oracle.py) against closed forms, the host stage of
inventory_from_grid against the oracle, the index -> network map against the sweep's fp32 grid points, the scene box's region
and its conversion to (scene_transform, extents), and manipulation_transform against the original's generate_poses_eval."""
import os
import sys

import numpy as np
import pytest

from dmnerf_b200 import objects as OB
from oracle import inventory_oracle as IO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXT = (1.9, 7.0, 7.0)


def _rot(ax, ay, az):
    cx, sx, cy, sy, cz, sz = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay), np.cos(az), np.sin(az)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def _transform(R=np.eye(3), t=(0.0, 0.0, 0.0)):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def _network_points(dim, T, ext=EXT):
    idx = np.stack(np.meshgrid(*[np.arange(dim)] * 3, indexing="ij"), -1).reshape(-1, 3)
    return IO.index_to_network(idx, T, dim, ext).reshape(dim, dim, dim, 3)


def _host_stage(occ, labels, T, ext, level, trim, n_labels):
    """inventory_from_grid's host stage fed with the oracle's integers and spans (what the two device passes return)."""
    dim = occ.shape[0]
    mom = np.zeros((n_labels, 10), dtype=np.int64)
    hist = np.zeros((n_labels, 3, dim), dtype=np.uint32)
    for g in range(n_labels):
        idx = IO.group_points(occ, labels, level, g)
        mom[g], hist[g] = IO.moments(idx), IO.histograms(idx, dim)
    boxes = OB.trimmed_boxes(hist, trim)
    obj = np.stack([IO.moments(IO.in_box(IO.group_points(occ, labels, level, g), boxes[g])) for g in range(n_labels)])
    A, b = OB.grid_affine(T, dim, ext)
    unit = abs(np.linalg.det(T[:3, :3])) * float(np.prod(np.asarray(ext) / (dim - 1)))
    entries, axes = OB.describe_groups(obj, boxes, A, b, unit, range(n_labels))
    spans = np.array([[IO.project(occ, labels, level, g, boxes[g], axes[g, r]) for r in range(3)] for g in range(n_labels)])
    return {e["label"]: e for e in OB.finish_obbs(entries, spans)}


# ------------------------------------------------------------------------------------------------- the oracle vs closed forms
def test_axis_aligned_box_count_centre_and_spans():
    dim = 40
    occ = np.zeros((dim,) * 3, np.float32)
    occ[5:15, 8:28, 3:10] = 1.0
    T = _transform(t=(0.3, -0.2, 0.5))
    e = IO.inventory(occ, None, T, EXT)[0]
    step = np.asarray(EXT) / (dim - 1)
    assert e["voxels"] == 10 * 20 * 7
    np.testing.assert_allclose(e["volume"], 1400 * np.prod(step), rtol=1e-14)
    mid = IO.index_to_network([[9.5, 17.5, 6.0]], T, dim, EXT)[0]
    np.testing.assert_allclose(e["centre"], mid, atol=1e-14)
    # index axes 1, 2, 0 (network z, -y, x) by decreasing length
    np.testing.assert_allclose(np.abs(e["obb"]["axes"]), [[0, 0, 1], [0, 1, 0], [1, 0, 0]], atol=1e-12)
    np.testing.assert_allclose(e["obb"]["half_sizes"], [19 * step[1] / 2, 6 * step[2] / 2, 9 * step[0] / 2], rtol=1e-12)
    lo, hi = e["aabb"]
    np.testing.assert_allclose(hi - lo, [9 * step[0], 6 * step[2], 19 * step[1]], rtol=1e-12)
    np.testing.assert_allclose(np.linalg.det(e["obb"]["axes"]), 1.0, atol=1e-12)


def test_rotated_box_obb_recovers_its_axes():
    dim = 96
    T = _transform(_rot(0.05, -0.04, 0.07), (0.1, 0.2, -0.3))
    p = _network_points(dim, T)
    Rb = _rot(0.6, 0.15, 0.1)                               # columns: the box's axes in the network frame
    c = IO.index_to_network([[47.5, 45.0, 49.0]], T, dim, EXT)[0]
    half = np.array([0.4, 2.0, 0.9])                         # the short axis lies along the grid's thin (1.9) side
    occ = np.all(np.abs((p - c) @ Rb) <= half, -1).astype(np.float32)
    e = IO.inventory(occ, None, T, EXT)[0]
    spacing = float(np.max(np.asarray(EXT) / (dim - 1)))
    for r, col in enumerate((1, 2, 0)):                      # descending extent
        assert abs(abs(e["obb"]["axes"][r] @ Rb[:, col]) - 1) < 2e-3, r
        assert abs(e["obb"]["half_sizes"][r] - half[col]) <= spacing, r
    np.testing.assert_allclose(e["obb"]["centre"], c, atol=spacing)


def test_ellipsoid_volume_centre_and_covariance():
    dim = 80
    T = _transform(t=(0.0, 0.4, 0.0))
    p = _network_points(dim, T)
    c = np.array([0.05, -0.3, 0.6])
    r = np.array([0.7, 2.1, 1.4])
    occ = (np.sum(((p - c) / r) ** 2, -1) <= 1).astype(np.float32)
    e = IO.inventory(occ, None, T, EXT)[0]
    np.testing.assert_allclose(e["volume"], 4 / 3 * np.pi * np.prod(r), rtol=0.03)
    np.testing.assert_allclose(e["centre"], c, atol=0.02)
    np.testing.assert_allclose(np.diag(e["covariance"]), r ** 2 / 5, rtol=0.05)
    np.testing.assert_allclose(np.sort(e["obb"]["half_sizes"])[::-1], np.sort(r)[::-1], atol=0.1)


def test_a_floater_is_removed_once_trim_exceeds_its_share():
    dim = 48
    occ = np.zeros((dim,) * 3, np.float32)
    occ[10:20, 12:22, 14:24] = 0.9
    only_box = IO.inventory(occ, None, np.eye(4), EXT)[0]
    occ[45, 2, 40] = 0.9                                                  # one voxel far away
    T = np.eye(4)
    untrimmed = IO.inventory(occ, None, T, EXT)[0]
    trimmed = IO.inventory(occ, None, T, EXT, trim=0.005)[0]              # floor(0.005 * 1001) = 5 points per end
    assert untrimmed["voxels"] == 1001 and trimmed["voxels"] == 1000
    assert np.all(untrimmed["aabb"][1] - untrimmed["aabb"][0] > only_box["aabb"][1] - only_box["aabb"][0] + 0.5)
    for k in ("centre", "covariance"):
        np.testing.assert_allclose(trimmed[k], only_box[k], rtol=0, atol=1e-15)
    np.testing.assert_array_equal(trimmed["box"], only_box["box"])
    np.testing.assert_allclose(trimmed["obb"]["half_sizes"], only_box["obb"]["half_sizes"], atol=1e-15)


# ------------------------------------------------------------------------------------------------- host stage vs the oracle
def _labelled_scene(dim, seed=0):
    g = np.random.default_rng(seed)
    T = _transform(_rot(0.1, 0.2, -0.3), (0.2, -0.1, 0.3))
    p = _network_points(dim, T)
    occ = (0.3 * g.random((dim,) * 3)).astype(np.float32)                  # below the level: background
    labels = np.full((dim,) * 3, 5, np.int16)
    sph = np.sum((p - [0.3, 1.5, 0.2]) ** 2, -1) <= 0.8 ** 2
    occ[sph], labels[sph] = 0.9, 1
    box = np.all(np.abs((p - [-0.2, -1.2, -1.0]) @ _rot(0.3, 0.1, 0.5)) <= [1.3, 0.6, 0.3], -1)
    occ[box], labels[box] = 0.8, 2
    edge = np.zeros_like(sph)
    edge[:, :4, :] = True                                                  # touches the grid boundary
    occ[edge], labels[edge] = 0.7, 3
    fl = g.integers(0, dim, (6, 3))
    occ[fl[:, 0], fl[:, 1], fl[:, 2]], labels[fl[:, 0], fl[:, 1], fl[:, 2]] = 0.95, 2   # floaters labelled as the box
    return occ, labels, T


@pytest.mark.parametrize("trim", [0.0, 0.004])
def test_host_stage_matches_the_oracle(trim):
    dim = 40
    occ, labels, T = _labelled_scene(dim)
    ours = _host_stage(occ, labels, T, EXT, 0.45, trim, 6)
    ref = IO.inventory(occ, labels, T, EXT, 0.45, trim, n_labels=6)
    assert sorted(ours) == sorted(ref) == [1, 2, 3]
    for g in ref:
        o, r = ours[g], ref[g]
        np.testing.assert_array_equal(o["box"], r["box"])
        assert o["voxels"] == r["voxels"]
        np.testing.assert_allclose(o["volume"], r["volume"], rtol=1e-14)
        np.testing.assert_allclose(o["centre"], r["centre"], rtol=0, atol=1e-13)
        np.testing.assert_allclose(o["covariance"], r["covariance"], rtol=0, atol=1e-12)
        for a, b in zip(o["aabb"], r["aabb"]):
            np.testing.assert_allclose(a, b, rtol=0, atol=1e-13)
        # spans are taken on our own axes: project the oracle's points on them
        idx = IO.in_box(IO.group_points(occ, labels, 0.45, g), r["box"])
        proj = (IO.index_to_network(idx, T, dim, EXT) - o["centre"]) @ o["obb"]["axes"].T
        np.testing.assert_allclose(o["obb"]["half_sizes"], (proj.max(0) - proj.min(0)) / 2, rtol=0, atol=1e-12)
        np.testing.assert_allclose(np.linalg.det(o["obb"]["axes"]), 1.0, atol=1e-12)


def test_trimmed_boxes_equal_the_sorted_coordinate_rule():
    dim = 32
    occ, labels, _ = _labelled_scene(dim, seed=3)
    hist = np.stack([IO.histograms(IO.group_points(occ, labels, 0.45, g), dim) for g in range(6)])
    for trim in (0.0, 0.001, 0.01, 0.1, 0.49):
        boxes = OB.trimmed_boxes(hist, trim)
        for g in range(6):
            idx = IO.group_points(occ, labels, 0.45, g)
            want = IO.trimmed_box(idx, trim) if idx.shape[0] else np.array([1, 0] * 3)
            np.testing.assert_array_equal(boxes[g], want, err_msg="label %d trim %g" % (g, trim))
    with pytest.raises(ValueError, match="trim"):
        OB._check_trim(0.5)


def test_affine_map_matches_the_sweeps_fp32_grid_points():
    g = np.random.default_rng(7)
    for dim in (2, 3, 64, 257):
        T = _transform(_rot(*g.uniform(-3, 3, 3)), g.uniform(-2, 2, 3))
        ext = g.uniform(0.5, 9, 3)
        idx = g.integers(0, dim, (500, 3))
        idx[:2] = [[0, 0, 0], [dim - 1, dim - 1, dim - 1]]
        A, b = OB.grid_affine(T, dim, ext)
        exact = idx @ A.T + b
        np.testing.assert_allclose(exact, IO.index_to_network(idx, T, dim, ext), rtol=0, atol=1e-14)
        fp32 = IO.grid_points_fp32(idx, T, dim, ext).astype(np.float64)
        scale = np.abs(T[:3, 3]).max() + np.abs(ext).max()
        assert np.abs(fp32 - exact).max() <= 4e-7 * scale, dim


def test_affine_map_rejects_a_reflection():
    T = np.diag([1.0, 1.0, -1.0, 1.0])
    with pytest.raises(ValueError, match="determinant"):
        OB.grid_affine(T, 8)


# ------------------------------------------------------------------------------------------------- the scene box on the host
def _cameras():
    from dmnerf_b200 import synth
    K = synth.dmsr_intrinsics(48, 64)
    poses = [synth.pose_spherical(th, -65.0, 7.0) for th in (0.0, 50.0, 130.0)]
    return poses, (48, 64, K)


def test_camera_region_holds_the_centres_and_the_far_corners():
    poses, (H, W, K) = _cameras()
    lo, hi = OB.camera_region(poses, (H, W, K), 15.0)
    from dmnerf_b200 import synth
    for c2w in poses:
        o, d = synth.rays_from_camera(H, W, K, c2w)
        for q in (0, W - 1, (H - 1) * W, H * W - 1):
            p = o[q].astype(np.float64) + 15.0 * d[q].astype(np.float64)
            assert np.all(p >= lo - 1e-5) and np.all(p <= hi + 1e-5)
        assert np.all(c2w[:3, 3] >= lo) and np.all(c2w[:3, 3] <= hi)


def test_region_and_box_transforms_round_trip_through_the_grid_points():
    poses, hwk = _cameras()
    lo, hi = OB.camera_region(poses, hwk, 15.0)
    T, ext = OB.region_transform(lo, hi)
    assert np.linalg.det(T[:3, :3]) == 1.0 and np.all(ext > 0)
    dim = 128
    corners = IO.grid_points_fp32([[0, 0, 0], [dim - 1, dim - 1, dim - 1]], T, dim, ext).astype(np.float64)
    pts = np.array([corners[0], corners[1]])
    np.testing.assert_allclose(pts.min(0), lo, rtol=0, atol=1e-5 * np.abs(hi - lo).max())
    np.testing.assert_allclose(pts.max(0), hi, rtol=0, atol=1e-5 * np.abs(hi - lo).max())
    box = np.array([7, 90, 0, 127, 33, 34])
    Tb, eb = OB.box_transform(T, ext, dim, box)
    assert np.linalg.det(Tb[:3, :3]) == 1.0
    sub = IO.grid_points_fp32([[0, 0, 0], [dim - 1, dim - 1, dim - 1]], Tb, dim, eb).astype(np.float64)
    parent = IO.grid_points_fp32([box[0::2], box[1::2]], T, dim, ext).astype(np.float64)
    np.testing.assert_allclose(sub, parent, rtol=0, atol=1e-5 * np.abs(hi - lo).max())


# ------------------------------------------------------------------------------------------------- manipulation transforms
def test_manipulation_transform_reproduces_the_original(golden_dir):
    g = np.load(os.path.join(golden_dir, "mani_transforms.npz"))
    assert len(g["scenes"]) == 8
    for scene in g["scenes"]:
        for mode in ("translation", "rotation", "scale", "multi"):
            d = OB.manipulation_transform(g[scene + "_centre"], mode)
            (entry,) = d["transformations"]
            assert entry["mode"] == mode
            np.testing.assert_array_equal(np.array(entry["transformation"]), g["%s_%s" % (scene, mode)], err_msg=scene + mode)
    with pytest.raises(ValueError, match="mode"):
        OB.manipulation_transform([0, 0, 0], "shear")


def test_find_objects_command_line():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import find_objects
    a = find_objects.parse(["ck.tar", "--poses", "p.npy", "--hwk", "48", "64", "32", "0", "31.5", "0", "32", "23.5", "0", "0", "1"])
    assert a.H == 48 and a.W == 64 and a.K.shape == (3, 3) and a.trim == 0.0
    a = find_objects.parse(["ck.tar", "--transform", "T.txt", "--extents", "1", "2", "3", "--trim", "0.01"])
    assert a.extents == [1.0, 2.0, 3.0] and a.trim == 0.01
    with pytest.raises(SystemExit):
        find_objects.parse(["ck.tar"])
    with pytest.raises(SystemExit):
        find_objects.parse(["ck.tar", "--poses", "p.npy"])


def test_extract_mesh_extents_option_defaults_to_the_original():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import extract_mesh
    assert extract_mesh.parse(["ck.tar", "T.npy", "--out", "o"]).extents == [1.9, 7.0, 7.0]
    assert extract_mesh.parse(["ck.tar", "T.npy", "--out", "o", "--extents", "2", "3", "4"]).extents == [2.0, 3.0, 4.0]
