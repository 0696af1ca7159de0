"""GPU: the object inventory -- the two device passes against the oracle's integers (oracle/inventory_oracle.py) on hand-made
labelled grids, their determinism and rejections; object_inventory on synthetic networks against the grid-only stage and the
per-object meshes; the scene box and extract_mesh over it; manipulator_eval about a found centre."""
import json
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from dmnerf_b200 import mesh as M
from dmnerf_b200 import objects as OB
from dmnerf_b200 import synth
from dmnerf_b200.engine import get_context
from dmnerf_b200.testing import make_models
from oracle import inventory_oracle as IO

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
EXT = (1.9, 7.0, 7.0)
N_LABELS = 8


def _rot(ax, ay, az):
    cx, sx, cy, sy, cz, sz = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay), np.cos(az), np.sin(az)
    return (np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
            @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]))


def _scene(dim, seed=0):
    """Labelled solids in a noisy background: two spheres, two rotated boxes, a slab touching the grid boundary, floaters
    labelled as one of the boxes; label 4 has no point, label 7 is the background."""
    g = np.random.default_rng(seed)
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = _rot(0.1, -0.2, 0.3), (0.2, -0.1, 0.3)
    idx = np.stack(np.meshgrid(*[np.arange(dim)] * 3, indexing="ij"), -1).reshape(-1, 3)
    p = IO.index_to_network(idx, T, dim, EXT).reshape(dim, dim, dim, 3)
    occ = (0.44 * g.random((dim,) * 3)).astype(np.float32)
    labels = np.full((dim,) * 3, 7, np.int16)

    def put(mask, value, lab):
        occ[mask], labels[mask] = value, lab
    put(np.sum((p - [0.3, 1.8, 0.2]) ** 2, -1) <= 0.7 ** 2, 0.9, 0)
    put(np.sum((p - [-0.2, -2.0, 1.6]) ** 2, -1) <= 0.45 ** 2, 0.6, 1)
    put(np.all(np.abs((p - [-0.1, -0.6, -1.5]) @ _rot(0.3, 0.1, 0.5)) <= [0.4, 1.4, 0.6], -1), 0.8, 2)
    put(np.all(np.abs((p - [0.1, 0.7, 1.9]) @ _rot(-0.4, 0.2, 0.9)) <= [0.3, 0.9, 0.5], -1), 0.7, 3)
    edge = np.zeros((dim,) * 3, bool)
    edge[:, :, : max(2, dim // 16)] = True
    put(edge, 0.99, 5)
    fl = g.integers(0, dim, (5, 3))
    occ[fl[:, 0], fl[:, 1], fl[:, 2]], labels[fl[:, 0], fl[:, 1], fl[:, 2]] = 0.95, 2
    labels[occ <= 0.45] = g.integers(0, N_LABELS, int((occ <= 0.45).sum()))      # background points carry any label
    return occ, labels, T


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.fixture(scope="module", params=[64, 256])
def scene(request):
    occ, labels, T = _scene(request.param)
    return occ, labels, T, _cu(occ), _cu(labels)


@pytest.mark.parametrize("with_labels", [True, False])
def test_voxels_equal_the_oracle_integers(scene, with_labels):
    occ, labels, T, d_occ, d_lab = scene
    lab, d_lab, n = (labels, d_lab, N_LABELS) if with_labels else (None, None, 1)
    dim = occ.shape[0]
    mom, hist = OB.object_voxels(d_occ, d_lab, 0.45, n)
    boxes = OB.trimmed_boxes(hist, 0.01)
    mom_b, _ = OB.object_voxels(d_occ, d_lab, 0.45, n, boxes)
    for g in range(n):
        idx = IO.group_points(occ, lab, 0.45, g)
        np.testing.assert_array_equal(mom[g], IO.moments(idx), err_msg="label %d" % g)
        np.testing.assert_array_equal(hist[g], IO.histograms(idx, dim), err_msg="label %d" % g)
        np.testing.assert_array_equal(mom_b[g], IO.moments(IO.in_box(idx, boxes[g])), err_msg="boxed label %d" % g)
        if idx.shape[0]:
            np.testing.assert_array_equal(boxes[g], IO.trimmed_box(idx, 0.01))
    if with_labels:
        assert mom[4, 0] == 0 and mom[5, 0] > 0


@pytest.mark.parametrize("trim", [0.0, 0.01])
def test_inventory_matches_the_oracle(scene, trim):
    occ, labels, T, d_occ, d_lab = scene
    dim = occ.shape[0]
    inv = OB.inventory_from_grid(d_occ, d_lab, T, EXT, 0.45, trim)
    ref = IO.inventory(occ, labels, T, EXT, 0.45, trim, n_labels=N_LABELS)
    assert [e["label"] for e in inv] == sorted(ref) == [0, 1, 2, 3, 5]
    A, b = OB.grid_affine(T, dim, EXT)
    for e in inv:
        r = ref[e["label"]]
        np.testing.assert_array_equal(e["box"], r["box"])
        assert e["voxels"] == r["voxels"]
        scale = np.abs(r["centre"]).max() + 1.0
        np.testing.assert_allclose(e["centre"], r["centre"], rtol=0, atol=1e-13 * scale)
        np.testing.assert_allclose(e["covariance"], r["covariance"], rtol=0, atol=1e-12 * np.abs(r["covariance"]).max())
        for a, c in zip(e["aabb"], r["aabb"]):
            np.testing.assert_allclose(a, c, rtol=0, atol=1e-13 * scale)
        # spans on the inventory's own axes: the oracle's points projected on them, in fp64
        idx = IO.in_box(IO.group_points(occ, labels, 0.45, e["label"]), r["box"])
        proj = (IO.index_to_network(idx, T, dim, EXT) - e["centre"]) @ e["obb"]["axes"].T
        extent = float(np.max(r["aabb"][1] - r["aabb"][0]))
        np.testing.assert_allclose(e["obb"]["half_sizes"], (proj.max(0) - proj.min(0)) / 2, rtol=0, atol=1e-9 * extent)
        # and bit for bit with the pass's own formula
        axes_in = np.concatenate([e["obb"]["axes"] @ A, (e["obb"]["axes"] @ (b - e["centre"]))[:, None]], 1)
        for q in range(3):
            lo, hi = IO.project(occ, labels, 0.45, e["label"], e["box"], axes_in[q])
            assert e["obb"]["half_sizes"][q] == (hi - lo) / 2
        np.testing.assert_allclose(np.linalg.det(e["obb"]["axes"]), 1.0, atol=1e-12)
    get_context(DEV).sync_check()


def test_two_calls_are_bit_identical(scene):
    _, _, T, d_occ, d_lab = scene
    a = OB.inventory_from_grid(d_occ, d_lab, T, EXT, 0.45, 0.01)
    b = OB.inventory_from_grid(d_occ, d_lab, T, EXT, 0.45, 0.01)
    m1, h1 = OB.object_voxels(d_occ, d_lab, 0.45, N_LABELS)
    m2, h2 = OB.object_voxels(d_occ, d_lab, 0.45, N_LABELS)
    assert np.array_equal(m1, m2) and np.array_equal(h1, h2)
    for x, y in zip(a, b):
        for k in ("centre", "covariance", "box"):
            assert np.array_equal(x[k], y[k]), k
        for k in ("centre", "axes", "half_sizes"):
            assert np.array_equal(x["obb"][k], y["obb"][k]), k


def test_rejections():
    dim = 16
    occ = torch.full((dim,) * 3, 0.9, device=DEV)
    labels = torch.zeros((dim,) * 3, device=DEV, dtype=torch.int16)
    boxes = np.tile([0, dim - 1] * 3, (4, 1))
    axes = np.zeros((4, 3, 4))
    bad = occ.clone()
    bad[3, 4, 5] = float("nan")
    with pytest.raises(RuntimeError, match="NaN"):
        OB.object_voxels(bad, labels, 0.45, 4)
    with pytest.raises(RuntimeError, match="NaN"):
        OB.object_spans(bad, labels, 0.45, 4, boxes, axes)
    lab = labels.clone()
    lab[1, 2, 3] = 4
    with pytest.raises(RuntimeError, match=r"label outside \[0, 3\]"):
        OB.object_voxels(occ, lab, 0.45, 4)
    with pytest.raises(RuntimeError, match=r"label outside \[0, 3\]"):
        OB.object_spans(occ, lab, 0.45, 4, boxes, axes)
    lab[1, 2, 3] = -1
    with pytest.raises(RuntimeError, match="label outside"):
        OB.object_voxels(occ, lab, 0.45, 4)
    for n in (0, 129):
        with pytest.raises(RuntimeError, match="n_labels %d out of range" % n):
            OB.object_voxels(occ, labels, 0.45, n)
    one = torch.ones((1, 1, 1), device=DEV)
    with pytest.raises(RuntimeError, match="dim 1 out of range"):
        OB.object_voxels(one, None, 0.45, 1)
    with pytest.raises(RuntimeError, match="dim 1 out of range"):
        OB.object_spans(one, None, 0.45, 1, np.zeros((1, 6)), np.zeros((1, 3, 4)))
    # the context stays usable
    mom, _ = OB.object_voxels(occ, labels, 0.45, 4)
    assert mom[0, 0] == dim ** 3


# ------------------------------------------------------------------------------------------------- synthetic networks
def _level(occ):
    """The synthetic networks need not cross 0.45: then the level leaves about 2% of the grid solid."""
    lo, hi = float(occ.min()), float(occ.max())
    if lo < 0.45 < hi and float((occ > 0.45).float().mean()) > 1e-3:
        return 0.45
    s = occ.flatten()[::7].float()
    return float(s.kthvalue(int(0.98 * s.numel())).values)


@pytest.mark.parametrize("ins_num", [13, 93])
def test_object_inventory_on_synthetic_networks(ins_num):
    nc, nf, _, _ = make_models(101, 202, ins_num, DEV)
    T = np.eye(4)
    T[:3, 3] = (0.1, -0.2, 0.3)
    dim = 96
    with torch.no_grad():
        occ, labels = OB.occupancy_objects(nf, T, OB.object_mask(ins_num, remove=[ins_num]), dim, device=DEV)
    level = _level(occ)
    inv = OB.object_inventory(nf, T, grid_dim=dim, level=level, trim=0.002)
    ref = OB.inventory_from_grid(occ, labels, T, None, level, 0.002, objects=range(ins_num))
    assert inv and len(inv) == len(ref)
    for a, b in zip(inv, ref):
        assert a["label"] == b["label"] and a["voxels"] == b["voxels"]
        for k in ("centre", "covariance", "box"):
            assert np.array_equal(a[k], b[k]), k
        assert np.array_equal(a["obb"]["half_sizes"], b["obb"]["half_sizes"])
    # every clean vertex of an object's mesh lies in its untrimmed AABB grown by one grid spacing
    full = {e["label"]: e for e in OB.inventory_from_grid(occ, labels, T, None, level, 0.0, objects=range(ins_num))}
    meshes = OB.meshes_from_labelled_grid(occ, labels, T, list(full), level, min_cluster=1)
    A, _ = OB.grid_affine(T, dim, M.EXTENTS)
    grow = np.abs(A).sum(1)
    checked = 0
    for k, m in meshes.items():
        v = m["clean_vertices"].cpu().double().numpy()
        net = np.stack([v[:, 0], -v[:, 2], v[:, 1]], -1)
        lo, hi = full[k]["aabb"]
        assert np.all(net >= lo - grow - 1e-5) and np.all(net <= hi + grow + 1e-5), k
        checked += v.shape[0]
    assert checked > 0
    get_context(DEV).sync_check()


def _checkpoint(tmp_path, ins_num=13):
    nc, nf, _, _ = make_models(101, 202, ins_num, "cpu")
    path = str(tmp_path / "ck.tar")
    torch.save({"network_coarse_state_dict": nc.state_dict(), "network_fine_state_dict": nf.state_dict()}, path)
    return path


def test_scene_box_and_extract_mesh_over_it(tmp_path):
    nc, nf, _, _ = make_models(101, 202, 13, DEV)
    H, W = 48, 64
    K = synth.dmsr_intrinsics(H, W)
    poses = np.stack([synth.pose_spherical(th, -65.0, 7.0) for th in (0.0, 60.0, 140.0, 250.0)])
    near, far = 4.0, 15.0
    lo, hi = OB.camera_region(poses, (H, W, K), far)
    T0, e0 = OB.region_transform(lo, hi)
    with torch.no_grad():
        occ = M.occupancy_grid(nf, T0, 64, e0, near, far, device=DEV)
    level = _level(occ)
    T, ext = OB.scene_box(nf, poses, (H, W, K), near, far, grid_dim=64, level=level)
    assert np.linalg.det(T[:3, :3]) == 1.0 and np.all(ext > 0)
    corners = np.array([[(ext / 2 * s) for s in (-1, 1)]]).reshape(2, 3) + T[:3, 3]
    net = np.stack([corners[:, 0], -corners[:, 2], corners[:, 1]], -1)
    tol = 1e-9 * float(np.abs(hi - lo).max())
    assert np.all(net.min(0) >= lo - tol) and np.all(net.max(0) <= hi + tol)
    out = M.extract_mesh(nf, nc, T, grid_dim=64, level=level, extents=tuple(ext), min_cluster=1)
    v = out["vertices"].cpu().double().numpy()
    assert v.shape[0] > 0
    local = v - T[:3, 3]
    assert np.all(np.abs(local) <= ext / 2 + 1e-5)
    # the command lines: find_objects writes the box, extract_mesh --extents uses it
    ck = _checkpoint(tmp_path)
    np.save(str(tmp_path / "poses.npy"), poses)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "find_objects.py"), ck, "--poses", str(tmp_path / "poses.npy"),
                        "--hwk", str(H), str(W)] + [repr(float(x)) for x in K.reshape(-1)] +
                       ["--level", repr(level), "--grid-dim", "48", "--box-grid-dim", "64", "--out", str(tmp_path / "box")],
                       capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    np.testing.assert_array_equal(np.array(res["scene_transform"]), T)
    np.testing.assert_array_equal(np.array(res["extents"]), ext)
    np.testing.assert_array_equal(np.loadtxt(str(tmp_path / "box" / "scene_transform.txt")), T)
    ext_txt = np.loadtxt(str(tmp_path / "box" / "extents.txt"))
    np.testing.assert_array_equal(ext_txt, ext)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "extract_mesh.py"), ck, str(tmp_path / "box" / "scene_transform.txt"),
                        "--extents"] + [repr(float(x)) for x in ext_txt] + ["--out", str(tmp_path / "mesh"), "--grid-dim", "48",
                                                                          "--min-cluster", "1"],
                       capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    ply = M.read_ply(str(tmp_path / "mesh" / "mesh.ply"))
    assert np.all(np.abs(ply["vertices"].astype(np.float64) - T[:3, 3]) <= ext / 2 + 1e-5)


def test_manipulator_eval_about_a_found_centre(tmp_path, monkeypatch):
    from dmnerf_b200.embedder import get_embedder
    from dmnerf_b200.manipulator import manipulator_eval
    ins_num = 13
    nc, nf, _, _ = make_models(101, 202, ins_num, DEV)
    T = np.eye(4)
    dim = 64
    with torch.no_grad():
        occ, _ = OB.occupancy_objects(nf, T, OB.object_mask(ins_num, remove=[ins_num]), dim, device=DEV)
    inv = OB.object_inventory(nf, T, grid_dim=dim, level=_level(occ))
    assert inv
    k = inv[0]["label"]
    trans = OB.manipulation_transform(inv[0]["centre"], "translation")
    (tmp_path / "data").mkdir()
    (tmp_path / "data" / "color_dict.json").write_text(json.dumps({"dmsr": {"study": {str(i): i for i in range(ins_num + 1)}}}))
    monkeypatch.chdir(tmp_path)
    H, W = 24, 32
    K = synth.dmsr_intrinsics(H, W)
    args = types.SimpleNamespace(datadir="./data/dmsr/study", device=torch.device(DEV), ins_num=ins_num, N_test=512, N_samples=64,
                                 N_importance=128, near=4.0, far=15.0, target_label=k)
    manipulator_eval(get_embedder(10)[0], get_embedder(4)[0], nc, nf, synth.pose_spherical(30.0, -65.0, 7.0)[None], (H, W, K), trans,
                     str(tmp_path / "out"), np.random.default_rng(0).integers(0, 256, (ins_num + 1, 3)), args)
    assert sorted(os.listdir(tmp_path / "out" / "translation")) == ["0_rgb.png"]
