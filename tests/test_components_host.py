"""CPU: the connected-components oracle on hand-made grids with known answers, and the host side of the component inventory:
the group look-up tables and their batches of 127, the largest-piece tie rule, the selection order, and find_objects.py's
flags and unchanged default output."""
import io
import json
import os
import sys
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

from dmnerf_b200 import objects as OB
from oracle import components_oracle as CO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import find_objects as FO          # noqa: E402


def _grid(dim, points, labels=None):
    occ = np.zeros((dim,) * 3, np.float32)
    lab = np.zeros((dim,) * 3, np.int16)
    for n, p in enumerate(points):
        occ[p] = 0.9
        if labels is not None:
            lab[p] = labels[n]
    return occ, lab


def test_diagonal_voxels_join_under_26_only():
    occ, _ = _grid(4, [(1, 1, 1), (2, 2, 2)])
    grid, label, voxels, root = CO.components(occ, None, 0.45, 26)
    assert voxels.tolist() == [2] and root.tolist() == [1 * 16 + 1 * 4 + 1]
    grid, label, voxels, root = CO.components(occ, None, 0.45, 6)
    assert voxels.tolist() == [1, 1] and root.tolist() == [21, 42]
    assert grid[1, 1, 1] == 0 and grid[2, 2, 2] == 1 and np.count_nonzero(grid >= 0) == 2
    occ, _ = _grid(4, [(1, 1, 1), (1, 2, 2)])                   # an edge neighbour
    assert CO.components(occ, None, 0.45, 6)[2].tolist() == [1, 1]
    assert CO.components(occ, None, 0.45, 26)[2].tolist() == [2]


def test_adjacent_voxels_with_different_labels_stay_apart():
    occ, lab = _grid(4, [(0, 0, 1), (0, 0, 2), (0, 0, 3)], [3, 5, 5])
    grid, label, voxels, root = CO.components(occ, lab, 0.45, 6)
    assert label.tolist() == [3, 5] and voxels.tolist() == [1, 2] and root.tolist() == [1, 2]
    assert grid[0, 0].tolist() == [-1, 0, 1, 1]
    # without labels they are one
    assert CO.components(occ, None, 0.45, 6)[2].tolist() == [3]


def test_a_non_solid_voxel_with_an_odd_label_is_ignored():
    occ, lab = _grid(4, [(0, 0, 0), (0, 0, 2)], [1, 1])
    lab[0, 0, 1] = 9                                            # between them, not solid
    occ[0, 0, 1] = 0.45                                         # occ > level is strict
    grid, label, voxels, root = CO.components(occ, lab, 0.45, 26)
    assert label.tolist() == [1, 1] and grid[0, 0, 1] == -1
    occ[0, 0, 1] = 0.46
    lab[0, 0, 1] = 1
    assert CO.components(occ, lab, 0.45, 26)[2].tolist() == [3]


def test_neighbours_do_not_wrap_across_a_face():
    dim = 5
    occ, _ = _grid(dim, [(2, 1, dim - 1), (2, 2, 0)])          # linear indices 59 and 60: consecutive, not neighbours
    assert np.ravel_multi_index((2, 2, 0), occ.shape) - np.ravel_multi_index((2, 1, dim - 1), occ.shape) == 1
    for conn in (6, 26):
        assert CO.components(occ, None, 0.45, conn)[2].tolist() == [1, 1]
    occ, _ = _grid(dim, [(1, dim - 1, 2), (2, 0, 2)])          # across the j face into the next plane
    for conn in (6, 26):
        assert CO.components(occ, None, 0.45, conn)[2].tolist() == [1, 1]


def test_hand_made_worst_cases():
    for dim in (5, 8):
        for conn in (6, 26):
            assert CO.components(CO.serpentine(dim), None, 0.45, conn)[2].shape == (1,)
        cb = CO.checkerboard(dim)
        assert CO.components(cb, None, 0.45, 6)[2].tolist() == [1] * int(cb.sum())
        assert CO.components(cb, None, 0.45, 26)[2].shape == (1,)


def test_numbering_is_by_smallest_linear_index():
    occ, lab = _grid(6, [(5, 5, 5), (0, 3, 0), (0, 3, 1), (2, 0, 0)], [0, 1, 1, 2])
    grid, label, voxels, root = CO.components(occ, lab, 0.45, 26)
    assert root.tolist() == sorted(root.tolist()) == [18, 72, 215]
    assert label.tolist() == [1, 2, 0] and voxels.tolist() == [2, 1, 1]


# ------------------------------------------------------------------------------------------------- host logic
def test_largest_component_tie_goes_to_the_smaller_root():
    label = np.array([4, 4, 2, 4, 2], np.int16)
    voxels = np.array([5, 7, 3, 7, 3])
    assert OB.largest_components(label, voxels) == {4: 1, 2: 2}
    assert OB.largest_components(label, voxels) == CO.largest(label, voxels, np.arange(5))
    assert OB.largest_components(np.zeros(0, np.int16), np.zeros(0)) == {}


def test_selection_order():
    label = np.array([3, 1, 3, 1, 0], np.int16)
    voxels = np.array([1, 5, 9, 2, 4])
    assert OB.select_components(label, voxels, "largest", range(4)) == [4, 1, 2]
    assert OB.select_components(label, voxels, "largest", [3]) == [2]
    assert OB.select_components(label, voxels, "split", range(4)) == [4, 1, 3, 0, 2]
    assert OB.select_components(label, voxels, "split", range(4), min_voxels=3) == [4, 1, 2]
    assert OB.select_components(label, voxels, "split", [1]) == [1, 3]


def test_group_luts_run_in_batches_of_127():
    assert OB.GROUP_BATCH == 127 and OB.DISCARD_GROUP == 127
    ids = list(range(300, 0, -1))                               # 300 components in entry order
    batches = OB.group_luts(ids, 301)
    assert [len(b) for _, b in batches] == [127, 127, 46]
    assert sum((b for _, b in batches), []) == ids
    for lut, batch in batches:
        assert lut.dtype == np.int16 and lut.shape == (301,)
        assert lut[batch].tolist() == list(range(len(batch)))
        rest = np.setdiff1d(np.arange(301), batch)
        assert np.all(lut[rest] == 127)
    assert OB.group_luts([], 5) == []


def test_inventory_argument_checks():
    with pytest.raises(ValueError, match="components must be"):
        OB.inventory_from_grid(torch.zeros(2, 2, 2), None, np.eye(4), components="all")
    with pytest.raises(ValueError, match="min_voxels"):
        OB.inventory_from_grid(torch.zeros(2, 2, 2), None, np.eye(4), components="largest", min_voxels=3)


# ------------------------------------------------------------------------------------------------- find_objects.py
def test_find_objects_flags():
    a = FO.parse(["ck.tar", "--transform", "T.txt"])
    assert a.components is None and FO.components_args(a) == {}
    a = FO.parse(["ck.tar", "--transform", "T.txt", "--components", "largest"])
    assert FO.components_args(a) == {"components": "largest", "connectivity": 26, "min_voxels": 1}
    a = FO.parse(["ck.tar", "--transform", "T.txt", "--components", "split", "--connectivity", "6", "--min-voxels", "9"])
    assert FO.components_args(a) == {"components": "split", "connectivity": 6, "min_voxels": 9}
    for bad in (["--connectivity", "18", "--components", "split"], ["--connectivity", "6"], ["--min-voxels", "3"],
                ["--components", "largest", "--min-voxels", "3"], ["--components", "whole"]):
        with pytest.raises(SystemExit):
            FO.parse(["ck.tar", "--transform", "T.txt"] + bad)


def _entry(**extra):
    e = {"label": 3, "voxels": 12, "volume": 0.25, "centre": np.array([0.1, -0.2, 0.3]),
         "aabb": (np.array([-1.0, -2.0, -3.0]), np.array([1.0, 2.0, 3.0])), "box": np.array([1, 2, 3, 4, 5, 6]),
         "covariance": np.eye(3), "obb": {"centre": np.array([0.0, 0.5, 1.0]), "axes": np.eye(3), "eigenvalues": np.ones(3),
                                          "half_sizes": np.array([0.5, 0.25, 0.125])}}
    e.update(extra)
    return e


def test_find_objects_default_output_is_unchanged(tmp_path, monkeypatch):
    from dmnerf_b200.testing import make_models
    nc, nf, _, _ = make_models(101, 202, 13, "cpu")
    ck = str(tmp_path / "ck.tar")
    torch.save({"network_coarse_state_dict": nc.state_dict(), "network_fine_state_dict": nf.state_dict()}, ck)
    np.savetxt(str(tmp_path / "T.txt"), np.eye(4))
    calls = []

    def fake(nf, T, ext, **kw):
        calls.append(kw)
        return [_entry()] if "components" not in kw else [_entry(components=2, discarded_voxels=5)]
    monkeypatch.setattr(OB, "object_inventory", fake)
    out = io.StringIO()
    with redirect_stdout(out):
        FO.main([ck, "--transform", str(tmp_path / "T.txt"), "--device", "cpu"])
    assert set(calls[0]) == {"grid_dim", "level", "trim", "near", "far", "N_importance"}
    e = _entry()
    want = {"scene_transform": np.eye(4).tolist(), "extents": [1.9, 7.0, 7.0], "trim": 0.0,
            "objects": [{"label": 3, "voxels": 12, "volume": 0.25, "centre": [0.1, -0.2, 0.3],
                         "aabb": [[-1.0, -2.0, -3.0], [1.0, 2.0, 3.0]],
                         "obb": {"centre": e["obb"]["centre"].tolist(), "axes": np.eye(3).tolist(),
                                 "half_sizes": [0.5, 0.25, 0.125]}}], "files": []}
    assert out.getvalue() == json.dumps(want) + "\n"
    out = io.StringIO()
    with redirect_stdout(out):
        FO.main([ck, "--transform", str(tmp_path / "T.txt"), "--device", "cpu", "--components", "largest"])
    assert calls[1]["components"] == "largest" and calls[1]["connectivity"] == 26
    got = json.loads(out.getvalue())["objects"][0]
    assert got["components"] == 2 and got["discarded_voxels"] == 5
    assert list(got)[:6] == ["label", "voxels", "volume", "centre", "aabb", "obb"]
