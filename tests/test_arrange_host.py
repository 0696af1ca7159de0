"""CPU: arranging objects -- the numpy restatement (oracle/arrange_oracle.py) on hand-built grids: the grid edit against the
edited-sweep oracle on grid points, a table moved and a box put on it, two boxes aimed at one point, an item that stays and blocks,
a spot freed by an earlier move, the object taken from the unedited grid under an obstacle mask; and the argument checks of the
Python layer and of the tool (no GPU)."""
import os
import sys

import numpy as np
import pytest
import torch

from dmnerf_b200 import objects as OB
from oracle import arrange_oracle as AO
from oracle import edit_sweep_oracle as E
from oracle import placement_oracle as PO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXT = (4.0, 4.0, 4.0)
DIM = 17                                             # grid points and 0.25 steps are exact in fp32
T = np.eye(4)
DOWN = (-1.0, 0.0, 0.0)                              # network -x = -e_i: height = index i
LEVEL = 0.45
FLOOR, TABLE, BOX, BOX2 = 6, 1, 2, 3


def _grid():
    occ, labels = np.zeros((DIM,) * 3, dtype=np.float32), np.zeros((DIM,) * 3, dtype=np.int16)
    occ[0], labels[0] = 0.9, FLOOR
    return occ, labels


def _put(occ, labels, box, label, value=0.9):
    occ[box], labels[box] = value, label


def _net(i, j, k):
    A, b = AO.grid_affine(T, DIM, EXT)
    return A @ np.array([i, j, k], dtype=np.float64) + b


def _solid(occ, labels, label):
    return (labels == label) & (occ > np.float32(LEVEL))


def _translate(d):
    A, _ = AO.grid_affine(T, DIM, EXT)
    m = np.eye(4)
    m[:3, 3] = -(A @ np.asarray(d, dtype=np.float64))
    return m


# ---- the grid edit --------------------------------------------------------------------------------------------------------------

def test_grid_edit_equals_the_edit_sweep_oracle_with_the_grid_as_network_on_grid_points():
    rng = np.random.default_rng(5)
    occ = rng.uniform(0.0, 1.0, (DIM,) * 3).astype(np.float32)
    labels = rng.integers(0, 4, (DIM,) * 3).astype(np.int16)
    inv, b = E.grid_index_map(T, EXT, DIM)
    turn = np.eye(4)
    turn[:3, :3] = [[1.0, 0.0, 0.0], [0.0, 0.0, -1.0], [0.0, 1.0, 0.0]]      # a quarter turn about x through the grid's centre
    moves = [{"label": 1, "trans": _translate((0, 2, -1)), "box": E.solid_box(occ, labels, 1, LEVEL, 0), "rest_drop": False},
             {"label": 2, "trans": turn, "box": E.solid_box(occ, labels, 2, LEVEL, 0), "rest_drop": False},
             {"label": 3, "trans": _translate((1, 0, 0)), "box": (2, 9, 3, 12, 0, 16), "rest_drop": False}]
    for n in (1, 3):
        o, l, landed, over = AO.grid_edit(occ, labels, occ, labels, T, EXT, moves[:n], LEVEL)
        want_o, want_l, _ = E.edit(occ, labels, T, EXT, moves[:n], E.grid_evaluate(occ, labels.astype(np.int64), inv, b), LEVEL)
        np.testing.assert_array_equal(o, want_o)
        np.testing.assert_array_equal(l, want_l)
        assert landed[0] > 0 and over[0].sum() > 0


def test_grid_edit_of_an_identity_or_an_absent_label_changes_nothing():
    occ, labels = _grid()
    _put(occ, labels, np.s_[1:3, 4:7, 4:7], BOX)
    for mv in ({"label": BOX, "trans": np.eye(4), "box": E.solid_box(occ, labels, BOX, LEVEL, 2)},
               {"label": 9, "trans": _translate((0, 3, 0)), "box": (0, DIM - 1) * 3}):
        o, l, landed, over = AO.grid_edit(occ, labels, occ, labels, T, EXT, [mv], LEVEL)
        np.testing.assert_array_equal(o, occ)
        np.testing.assert_array_equal(l, labels)
        assert over.sum() == 0


# ---- hand-built arrangements ----------------------------------------------------------------------------------------------------

def _table_scene():
    """A floor, a table (label 1: a top at i 4 on four legs) in one corner and a box (label 2) in the other."""
    occ, labels = _grid()
    _put(occ, labels, np.s_[4, 1:6, 1:6], TABLE)
    for j in (1, 5):
        for k in (1, 5):
            _put(occ, labels, np.s_[1:4, j, k], TABLE)
    _put(occ, labels, np.s_[1:3, 12:14, 12:14], BOX)
    return occ, labels


def test_a_moved_table_carries_a_box_put_on_it():
    occ, labels = _table_scene()
    items = [{"label": TABLE, "near": _net(0, 10, 4)}, {"label": BOX, "near": _net(0, 10, 4), "on": [TABLE], "lift": 4}]
    o, l, chosen = AO.arrange(occ, labels, T, EXT, items, DOWN, LEVEL)
    assert all(c is not None for c in chosen)
    table, box = _solid(o, l, TABLE), _solid(o, l, BOX)
    assert table.sum() == _solid(occ, labels, TABLE).sum() and box.sum() == _solid(occ, labels, BOX).sum()
    top = np.argwhere(table)[:, 0].max()
    bi = np.argwhere(box)
    assert bi[:, 0].min() == top + 1                               # on the table's new top
    assert all(table[top, j, k] for _, j, k in bi)
    assert not table[4, 1:6, 1:6].all()                            # the table left its corner


def test_two_boxes_aimed_at_one_point_do_not_overlap():
    occ, labels = _grid()
    _put(occ, labels, np.s_[1:3, 1:3, 1:3], BOX)
    _put(occ, labels, np.s_[1:3, 13:15, 13:15], BOX2)
    aim = _net(0, 8, 8)
    o, l, chosen = AO.arrange(occ, labels, T, EXT, [{"label": BOX, "near": aim}, {"label": BOX2, "near": aim}], DOWN, LEVEL)
    assert all(c is not None for c in chosen)
    a, b = _solid(o, l, BOX), _solid(o, l, BOX2)
    assert a.sum() == 8 and b.sum() == 8 and not (a & b).any()
    assert chosen[0]["offset"] != chosen[1]["offset"]


def test_an_item_that_cannot_be_placed_stays_and_blocks_a_later_one():
    occ, labels = _grid()
    _put(occ, labels, np.s_[1:3, 7:10, 7:10], BOX)                 # stays: nothing of label 5 to rest on
    _put(occ, labels, np.s_[1:3, 1:3, 1:3], BOX2)
    items = [{"label": BOX, "near": _net(0, 2, 2), "on": [5]}, {"label": BOX2, "near": _net(0, 8, 8), "on": [FLOOR]}]
    o, l, chosen = AO.arrange(occ, labels, T, EXT, items, DOWN, LEVEL)
    assert chosen[0] is None and chosen[1] is not None
    np.testing.assert_array_equal(_solid(o, l, BOX), _solid(occ, labels, BOX))
    assert not (_solid(o, l, BOX2) & _solid(occ, labels, BOX)).any()


def test_a_spot_is_taken_only_after_the_item_standing_there_moved():
    occ, labels = _grid()
    _put(occ, labels, np.s_[1:3, 7:10, 7:10], BOX)
    _put(occ, labels, np.s_[1:3, 1:4, 1:4], BOX2)
    spot = _net(0, 8, 8)
    alone = AO.arrange(occ, labels, T, EXT, [{"label": BOX2, "near": spot, "on": [FLOOR]}], DOWN, LEVEL)
    both = AO.arrange(occ, labels, T, EXT, [{"label": BOX, "near": _net(0, 14, 14)}, {"label": BOX2, "near": spot, "on": [FLOOR]}],
                      DOWN, LEVEL)
    assert both[2][1]["offset"] == (6, 6)                           # exactly where BOX stood
    assert alone[2][0]["offset"] != (6, 6)
    np.testing.assert_array_equal(_solid(both[0], both[1], BOX2), _solid(occ, labels, BOX))


def test_an_obstacle_mask_lets_an_item_land_over_a_later_one_which_is_still_placed_whole():
    occ, labels = _grid()
    _put(occ, labels, np.s_[1:3, 2:5, 2:5], BOX)
    _put(occ, labels, np.s_[1:3, 8:11, 8:11], BOX2)
    items = [{"label": BOX, "near": _net(0, 9, 9), "obstacles": [FLOOR]}, {"label": BOX2, "near": _net(0, 3, 14)}]
    axis, sign = PO.down_axis(T, EXT, DOWN)
    o, l, chosen = AO.arrange(occ, labels, T, EXT, items[:1], DOWN, LEVEL)
    assert chosen[0]["offset"] == (6, 6) and (_solid(o, l, BOX2).sum() < 18)     # BOX landed over part of BOX2
    box = E.solid_box(occ, labels, BOX2, LEVEL, 2)
    m = AO.placement_in_scene(occ, labels, o, l, T, EXT, BOX2, LEVEL, axis, sign, 0, np.eye(4), box)
    assert m["points"].shape[0] == 18                              # from the unedited grid: whole
    o2, l2, chosen = AO.arrange(occ, labels, T, EXT, items, DOWN, LEVEL)
    assert chosen[1] is not None and _solid(o2, l2, BOX2).sum() == 18


# ---- argument checks --------------------------------------------------------------------------------------------------------------

def test_python_layer_rejects_bad_items_before_any_device_work():
    occ, labels = torch.zeros((DIM,) * 3), torch.zeros((DIM,) * 3, dtype=torch.int16)
    ok = {"label": 1, "near": (0.0, 0.0, 0.0)}
    bad = [[], [dict(ok, colour=3)], [{"near": (0, 0, 0)}], [{"label": 1}], [ok, dict(ok)], [dict(ok, label=k) for k in range(9)],
           [dict(ok, label=128)], [dict(ok, near=(0, 0))], [dict(ok, on=[200])], [dict(ok, turns=0)], [dict(ok, stable=1)],
           [dict(ok, lift=-1)], [dict(ok, lift=DIM)], [dict(ok, lift=1.5)], [dict(ok, rest="away")], [dict(ok, obstacles=[300])],
           [dict(ok, piece="cube")], [5], {"label": 1, "near": (0, 0, 0)}]
    for items in bad:
        with pytest.raises(ValueError):
            OB.arrange_objects(occ, labels, T, items, DOWN, EXT)
    for kw in ({"max_tests": 0}, {"level": 1.5}):
        with pytest.raises(ValueError):
            OB.arrange_objects(occ, labels, T, [ok], DOWN, EXT, **kw)
    with pytest.raises(ValueError):
        OB.arrange_objects(occ, labels, T, [ok], (0.0, 0.0, 0.0), EXT)


def test_tool_rejects_arrange_with_a_single_move_flag(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import move_objects
    spec = tmp_path / "spec.json"
    spec.write_text('[{"label": 1, "near": [0, 0, 0]}]')
    base = ["ck.tar", "--pose", "p.npy", "--hwk", "4", "4"] + ["1"] * 9 + ["--transform", "t.npy", "--out", "o"]
    a = move_objects.parse(base + ["--arrange", str(spec), "--down", "0", "-1", "0"])
    assert a.arrange == str(spec) and a.move_label is None
    for extra in (["--place-at", "0", "0", "0"], ["--mode", "translation"], ["--until-contact"], ["--distance", "1"],
                  ["--yaw", "30"], ["--scale", "2"], ["--turns", "4"], ["--move-label", "1"]):
        with pytest.raises(SystemExit):
            move_objects.parse(base + ["--arrange", str(spec), "--down", "0", "-1", "0"] + extra)
    with pytest.raises(SystemExit):                                # --arrange needs --down
        move_objects.parse(base + ["--arrange", str(spec)])
