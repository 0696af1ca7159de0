"""GPU: connected components -- the id grid and the per-component table against scipy (oracle/components_oracle.py), bit for
bit, on the inventory test's labelled scene and on hand-made worst cases; determinism and rejections; the inventory and the
per-object meshes restricted to components, against the inventory oracle and marching cubes of the masked field; the
synthetic networks and find_objects --components."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from dmnerf_b200 import _lib
from dmnerf_b200 import mesh as M
from dmnerf_b200 import objects as OB
from dmnerf_b200.engine import get_context
from dmnerf_b200.testing import make_models
from oracle import components_oracle as CO
from oracle import inventory_oracle as IO
from test_gpu_inventory import EXT, _level, _scene

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


_SCENES = {}


def scene(dim):
    if dim not in _SCENES:
        _SCENES[dim] = _scene(dim)
    return _SCENES[dim]


def _check(occ, labels, conn):
    got = OB.object_components(_cu(occ), None if labels is None else _cu(labels), 0.45, conn)
    grid, label, voxels, root = CO.components(occ, labels, 0.45, conn)
    assert np.array_equal(got["grid"].cpu().numpy(), grid)
    assert np.array_equal(got["label"], label) and got["label"].dtype == np.int16
    assert np.array_equal(got["voxels"], voxels) and np.array_equal(got["root"], root)
    return got


@pytest.mark.parametrize("dim", [64, 97, 256])
@pytest.mark.parametrize("conn", [6, 26])
@pytest.mark.parametrize("with_labels", [True, False])
def test_scene_equals_the_oracle(dim, conn, with_labels):
    occ, labels, _ = scene(dim)
    got = _check(occ, labels if with_labels else None, conn)
    if with_labels:
        assert np.count_nonzero(got["label"] == 2) >= 2            # box 2 and its floaters
    get_context(DEV).sync_check()


@pytest.mark.parametrize("kind", ["serpentine", "checkerboard", "full", "empty"])
@pytest.mark.parametrize("conn", [6, 26])
@pytest.mark.parametrize("dim", [97, 256])
def test_hand_made_grids(kind, conn, dim):
    occ = {"serpentine": CO.serpentine, "checkerboard": CO.checkerboard,
           "full": lambda d: np.ones((d,) * 3, np.float32), "empty": lambda d: np.zeros((d,) * 3, np.float32)}[kind](dim)
    got = _check(occ, None, conn)
    n = got["voxels"].shape[0]
    expect = {"serpentine": 1, "full": 1, "empty": 0,
              "checkerboard": int(np.count_nonzero(occ)) if conn == 6 else 1}[kind]
    assert n == expect


def test_two_calls_are_bit_identical():
    occ, labels, _ = scene(256)
    for o, lab in ((occ, labels), (CO.serpentine(256), None)):
        a = OB.object_components(_cu(o), None if lab is None else _cu(lab), 0.45, 26)
        b = OB.object_components(_cu(o), None if lab is None else _cu(lab), 0.45, 26)
        assert torch.equal(a["grid"], b["grid"])
        for k in ("label", "voxels", "root"):
            assert np.array_equal(a[k], b[k]), k


def test_rejections():
    dim = 16
    occ = torch.full((dim,) * 3, 0.9, device=DEV)
    labels = torch.zeros((dim,) * 3, device=DEV, dtype=torch.int16)
    bad = occ.clone()
    bad[3, 4, 5] = float("nan")
    with pytest.raises(RuntimeError, match="NaN"):
        OB.object_components(bad, labels)
    lab = labels.clone()
    lab[1, 2, 3] = 128
    with pytest.raises(RuntimeError, match=r"label outside \[0, 127\]"):
        OB.object_components(occ, lab)
    with pytest.raises(RuntimeError, match="connectivity 18 is not 6 or 26"):
        OB.object_components(occ, labels, connectivity=18)
    # dim 1291: rejected on the host before any launch, so small buffers stand in for the grids
    ctx = get_context(DEV)
    comp = torch.empty((dim,) * 3, dtype=torch.int32, device=DEV)
    n = C.c_int64(-7)
    with pytest.raises(RuntimeError, match="dim 1291 out of range"):
        ctx.call("dmnerf_object_components", ctx.handle, _lib.ptr(occ), None, 1291, 0.45, 1, 26, _lib.ptr(comp, torch.int32),
                 C.byref(n))
    assert n.value == -7
    # a component id outside [-1, n) in the id grid
    ids = torch.full((dim,) * 3, 5, dtype=torch.int32, device=DEV)
    with pytest.raises(RuntimeError, match="id outside"):
        OB.component_groups(ids, np.zeros(3, np.int16), 127)
    # the context stays usable
    got = OB.object_components(occ, labels)
    assert got["voxels"].tolist() == [dim ** 3] and got["root"].tolist() == [0]
    ctx.sync_check()


# ------------------------------------------------------------------------------------------------- inventory and meshes
def _same_entry(e, r, dim):
    np.testing.assert_array_equal(e["box"], r["box"])
    assert e["voxels"] == r["voxels"]
    scale = np.abs(r["centre"]).max() + 1.0
    np.testing.assert_allclose(e["centre"], r["centre"], rtol=0, atol=1e-13 * scale)
    np.testing.assert_allclose(e["covariance"], r["covariance"], rtol=0, atol=1e-12 * np.abs(r["covariance"]).max())
    for a, c in zip(e["aabb"], r["aabb"]):
        np.testing.assert_allclose(a, c, rtol=0, atol=1e-13 * scale)
    extent = float(np.max(r["aabb"][1] - r["aabb"][0])) + 1e-12
    np.testing.assert_allclose(e["obb"]["half_sizes"], r["obb"]["half_sizes"], rtol=0, atol=1e-9 * extent)


def _masked_inventory(occ, mask, T, trim):
    return IO.inventory(np.where(mask, occ, np.float32(0)), None, T, EXT, 0.45, trim, n_labels=1)[0]


@pytest.mark.parametrize("dim", [64, 97])
@pytest.mark.parametrize("trim", [0.0, 0.01])
@pytest.mark.parametrize("conn", [6, 26])
def test_largest_equals_the_oracle_of_the_masked_grid(dim, trim, conn):
    occ, labels, T = scene(dim)
    inv = OB.inventory_from_grid(_cu(occ), _cu(labels), T, EXT, 0.45, trim, components="largest", connectivity=conn)
    grid, label, voxels, root = CO.components(occ, labels, 0.45, conn)
    best = CO.largest(label, voxels, root)
    assert [e["label"] for e in inv] == sorted(best) == [0, 1, 2, 3, 5]
    for e in inv:
        k = e["label"]
        _same_entry(e, _masked_inventory(occ, grid == best[k], T, trim), dim)
        assert e["components"] == int(np.count_nonzero(label == k))
        assert e["discarded_voxels"] == int(voxels[label == k].sum() - voxels[best[k]])
    box2 = next(e for e in inv if e["label"] == 2)
    assert box2["components"] >= 2 and box2["discarded_voxels"] >= 1       # the floaters are gone


@pytest.mark.parametrize("min_voxels", [1, 3])
def test_split_equals_the_per_component_oracle(min_voxels):
    dim = 64
    occ, labels, T = scene(dim)
    inv = OB.inventory_from_grid(_cu(occ), _cu(labels), T, EXT, 0.45, 0.0, components="split", min_voxels=min_voxels)
    grid, label, voxels, root = CO.components(occ, labels, 0.45, 26)
    want = sorted([c for c in range(len(label)) if voxels[c] >= min_voxels], key=lambda c: (int(label[c]), int(root[c])))
    assert [(e["label"], e["component"]) for e in inv] == [(int(label[c]), c) for c in want]
    for e in inv:
        _same_entry(e, _masked_inventory(occ, grid == e["component"], T, 0.0), dim)


def test_split_runs_in_batches_of_127():
    dim = 16
    occ = CO.checkerboard(dim)                                  # 2048 one-voxel components under 6-connectivity
    T = np.eye(4)
    inv = OB.inventory_from_grid(_cu(occ), None, T, EXT, 0.45, components="split", connectivity=6)
    assert [e["component"] for e in inv] == list(range(int(np.count_nonzero(occ))))
    A, b = OB.grid_affine(T, dim, EXT)
    flat = np.nonzero(occ.reshape(-1))[0]
    for e in inv[::97]:
        idx = np.array(np.unravel_index(flat[e["component"]], occ.shape), np.float64)
        np.testing.assert_allclose(e["centre"], A @ idx + b, rtol=0, atol=1e-12)
        assert e["voxels"] == 1


def test_components_none_is_todays_call():
    occ, labels, T = scene(64)
    a = OB.inventory_from_grid(_cu(occ), _cu(labels), T, EXT, 0.45, 0.01)
    b = OB.inventory_from_grid(_cu(occ), _cu(labels), T, EXT, 0.45, 0.01, components=None, connectivity=6, min_voxels=1)
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert set(x) == set(y) and "components" not in x and "component" not in x
        for k in ("label", "voxels", "volume"):
            assert x[k] == y[k]
        for k in ("centre", "covariance", "box"):
            assert np.array_equal(x[k], y[k]), k
        for k in ("centre", "axes", "half_sizes"):
            assert np.array_equal(x["obb"][k], y["obb"][k]), k


def test_object_meshes_of_the_largest_component():
    ins_num = 13
    nc, nf, _, _ = make_models(101, 202, ins_num, DEV)
    T = np.eye(4)
    dim = 64
    with torch.no_grad():
        occ, labels = OB.occupancy_objects(nf, T, OB.object_mask(ins_num, remove=[ins_num]), dim, device=DEV)
    level = _level(occ)
    got = OB.object_meshes(nf, nc, T, grid_dim=dim, level=level, min_cluster=1, components="largest")
    o, lab = occ.cpu().numpy(), labels.cpu().numpy()
    grid, label, voxels, root = CO.components(o, lab, level, 26)
    best = CO.largest(label, voxels, root)
    objects = [k for k in np.unique(lab).tolist() if k != ins_num]
    assert sorted(got) == objects
    for k in objects:
        field = torch.where(_cu(grid) == best[k], occ, torch.zeros((), device=DEV)) if k in best else torch.zeros_like(occ)
        v, t = M.marching_cubes(field, level)
        assert torch.equal(M.to_scene(v, T, dim, M.EXTENTS), got[k]["vertices"]), k
        assert torch.equal(t, got[k]["triangles"]), k
    get_context(DEV).sync_check()


@pytest.mark.parametrize("ins_num", [13, 93])
def test_object_inventory_on_synthetic_networks(ins_num):
    """Where a label has one component the largest-component entry is the unsplit one; every entry is the unsplit inventory
    of the sweep masked to its component."""
    nc, nf, _, _ = make_models(101, 202, ins_num, DEV)
    T = np.eye(4)
    T[:3, 3] = (0.1, -0.2, 0.3)
    dim = 96
    with torch.no_grad():
        occ, labels = OB.occupancy_objects(nf, T, OB.object_mask(ins_num, remove=[ins_num]), dim, device=DEV)
    level = _level(occ)
    whole = {e["label"]: e for e in OB.object_inventory(nf, T, grid_dim=dim, level=level, trim=0.002)}
    largest = OB.object_inventory(nf, T, grid_dim=dim, level=level, trim=0.002, components="largest")
    assert largest and sorted(e["label"] for e in largest) == sorted(whole)
    cc = OB.object_components(occ, labels, level, 26)
    best = OB.largest_components(cc["label"], cc["voxels"])
    zero = torch.zeros((), device=DEV)
    for e in largest:
        refs = [OB.inventory_from_grid(torch.where(cc["grid"] == best[e["label"]], occ, zero), None, T, None, level, 0.002)[0]]
        if e["components"] == 1:
            assert e["discarded_voxels"] == 0
            refs.append(whole[e["label"]])
        for w in refs:
            assert e["voxels"] == w["voxels"]
            for k in ("centre", "covariance", "box"):
                assert np.array_equal(e[k], w[k]), k
            assert np.array_equal(e["obb"]["half_sizes"], w["obb"]["half_sizes"])


def test_find_objects_with_components(tmp_path):
    ins_num = 13
    nc, nf, _, _ = make_models(101, 202, ins_num, "cpu")
    ck = str(tmp_path / "ck.tar")
    torch.save({"network_coarse_state_dict": nc.state_dict(), "network_fine_state_dict": nf.state_dict()}, ck)
    T = np.eye(4)
    np.savetxt(str(tmp_path / "T.txt"), T)
    dim = 48
    nf = nf.to(DEV)
    with torch.no_grad():
        occ, _ = OB.occupancy_objects(nf, T, OB.object_mask(ins_num, remove=[ins_num]), dim, device=DEV)
    level = _level(occ)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "find_objects.py"), ck, "--transform", str(tmp_path / "T.txt"),
                        "--grid-dim", str(dim), "--level", repr(level), "--components", "largest", "--connectivity", "6"],
                       capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    want = OB.object_inventory(nf, T, grid_dim=dim, level=level, components="largest", connectivity=6)
    assert res["objects"] and len(res["objects"]) == len(want)
    for o, e in zip(res["objects"], want):
        assert (o["label"], o["voxels"], o["components"], o["discarded_voxels"]) == (e["label"], e["voxels"], e["components"],
                                                                                  e["discarded_voxels"])
        assert o["centre"] == e["centre"].tolist()
