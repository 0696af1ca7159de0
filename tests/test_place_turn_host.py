"""CPU: turned placements -- the numpy restatement (oracle/placement_turn_oracle.py) on hand-built grids: quarter turns against
numpy index rotations, a bar that only passes a slot when turned, the identity base, the exact turn matrices, turns that do not
fit, the order of candidates across turns, and the argument checks of the Python layer and of the tools (no GPU)."""
import os
import sys
from fractions import Fraction

import numpy as np
import pytest
import torch

from dmnerf_b200 import objects as OB
from oracle import edit_sweep_oracle as E
from oracle import placement_oracle as PO
from oracle import placement_turn_oracle as TO
from oracle import region_oracle as RO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXT = (4.0, 4.0, 4.0)
DIM = 17                                             # grid points and 0.25 steps are exact in fp32
T = np.eye(4)
UP_I = (-1.0, 0.0, 0.0)                              # network -x = -e_i: height = index i, turns about e_i


def _grid():
    return np.zeros((DIM,) * 3, dtype=np.float32), np.zeros((DIM,) * 3, dtype=np.int16)


def _put(occ, labels, box, label, value=0.9):
    occ[box], labels[box] = value, label


def _extent(occ, labels, label):
    mask = torch.from_numpy((labels == label) & (occ > np.float32(0.45)))
    return OB._object_extent(mask)


def _turned(occ, labels, label, angle, down=UP_I, lift=0, **kw):
    """The oracle map of `label` turned by `angle` -> (map, base), base None when the turn does not fit."""
    axis, sign = PO.down_axis(T, EXT, down)
    _, box, centre = _extent(occ, labels, label)
    (a, base), = OB.turn_bases(T, DIM, axis, centre, box, [angle], EXT)
    want = TO.turn_base(T, EXT, DIM, axis, centre, box, angle)
    assert (base is None) == (want is None)
    if base is None:
        return None, None
    np.testing.assert_array_equal(base, want)
    src = E.solid_box(occ, labels, label, 0.45, 2)
    return TO.placement_map(occ, labels, T, EXT, label, 0.45, axis, sign, lift, base, src, **kw), base


def _scene(rng):
    """A floor (label 6) at i 0, random blocks of labels 2..5, and an L-shape (label 1) at i 12..13."""
    occ, labels = _grid()
    _put(occ, labels, np.s_[0], 6)
    for _ in range(14):
        a, b, c = rng.integers(1, 8), rng.integers(0, DIM - 3), rng.integers(0, DIM - 3)
        _put(occ, labels, np.s_[a:a + 3, b:b + 2, c:c + 3], int(rng.integers(2, 6)))
    _put(occ, labels, np.s_[12:14, 5:10, 7], 1)
    _put(occ, labels, np.s_[12:14, 5, 8:11], 1)
    return occ, labels


def test_quarter_turns_of_an_l_shape_equal_the_l_rotated_by_index_permutation():
    occ, labels = _scene(np.random.default_rng(3))
    for k in (1, 2, 3):
        m, _ = _turned(occ, labels, 1, 90.0 * k)
        # the same L rotated in the (j, k) plane by numpy: a turn by +90 degrees about +e_i carries +e_j to +e_k
        rot_occ, rot_lab = occ.copy(), labels.copy()
        L = (labels == 1)
        rot_occ[L], rot_lab[L] = 0.0, 0
        turned = np.rot90(L, k, axes=(1, 2))
        rot_occ[turned], rot_lab[turned] = 0.9, 1
        assert not ((labels[turned] != 0) & (labels[turned] != 1)).any()
        axis, sign = PO.down_axis(T, EXT, UP_I)
        want = PO.placement_map(rot_occ, rot_lab, T, EXT, 1, 0.45, axis, sign, 0)
        for key in ("drop", "contacts", "support"):
            np.testing.assert_array_equal(m[key], want[key], err_msg="%s at %d degrees" % (key, 90 * k))
        assert len(np.unique(m["drop"])) > 2 and len(np.unique(m["support"])) > 2
        assert m["points"].shape[0] == 16                                  # nothing clipped, nothing resampled


def test_a_bar_rests_on_the_walls_unturned_and_drops_through_the_slot_turned():
    occ, labels = _grid()
    _put(occ, labels, np.s_[0:2], 3)                                   # floor
    _put(occ, labels, np.s_[2:9], 2)                                   # two walls ...
    occ[2:9, 8, :], labels[2:9, 8, :] = 0.0, 0                          # ... with a slot one voxel wide along k
    _put(occ, labels, np.s_[12, 7:10, 4], 1)                           # a 1 x 3 bar along j
    m0, _ = _turned(occ, labels, 1, 0.0)
    assert (m0["drop"] == 3).all() and (m0["support"] == 2).all()        # onto the walls' top at i 8
    m90, base = _turned(occ, labels, 1, 90.0)
    assert (m90["drop"] >= 3).all() and int(m90["drop"].max()) == 10 and int((m90["drop"] == 10).sum()) == DIM - 2
    assert set(np.unique(m90["support"][m90["drop"] == 10]).tolist()) == {3}
    assert m90["drop"].shape == (DIM, DIM - 2)                           # 1 wide along j, 3 long along k


def test_the_identity_base_equals_the_unturned_map():
    occ, labels = _scene(np.random.default_rng(8))
    axis, sign = PO.down_axis(T, EXT, UP_I)
    src = E.solid_box(occ, labels, 1, 0.45, 2)
    for lift in (0, 2):
        want = PO.placement_map(occ, labels, T, EXT, 1, 0.45, axis, sign, lift)
        got = TO.placement_map(occ, labels, T, EXT, 1, 0.45, axis, sign, lift, np.eye(4), src)
        for key in ("drop", "contacts", "support"):
            np.testing.assert_array_equal(got[key], want[key])
        assert got["centre"] == want["centre"] and got["offset_lo"] == want["offset_lo"]
    mask = np.zeros((DIM,) * 3, dtype=bool)
    mask[12:14, 5:8] = True
    A, b = OB.grid_affine(T, DIM, EXT)
    piece = E.Piece(RO.pack(mask), DIM, RO.voxel_map(A, b), outside_keep=False)
    for rest in (False, True):
        want = PO.placement_map(occ, labels, T, EXT, 1, 0.45, axis, sign, 0, piece, rest)
        got = TO.placement_map(occ, labels, T, EXT, 1, 0.45, axis, sign, 0, np.eye(4), src, piece, rest)
        for key in ("drop", "contacts", "support"):
            np.testing.assert_array_equal(got[key], want[key])


def test_quarter_turn_bases_are_exact_and_other_angles_are_rotations():
    A, _ = OB.grid_affine(T, DIM, EXT)
    for axis in range(3):
        for angle in (0, 90, 180, 270, -90, 450, 45.0, 20.0):
            (a, base), = OB.turn_bases(T, DIM, axis, [Fraction(8)] * 3, (6, 10) * 3, [angle], EXT)
            R = base[:3, :3]
            np.testing.assert_allclose(R @ R.T, np.eye(3), rtol=0, atol=1e-15)
            assert np.linalg.det(R) > 0 and a == float(angle)
            n = A[:, axis] / np.linalg.norm(A[:, axis])
            np.testing.assert_allclose(R @ n, n, rtol=0, atol=1e-15)           # about the down index axis
            if float(angle) % 90 == 0:
                assert set(np.unique(R).tolist()) <= {-1.0, 0.0, 1.0}
                np.testing.assert_array_equal(base, TO.turn_base(T, EXT, DIM, axis, [8, 8, 8], (6, 10) * 3, angle))
    (_, b90), = OB.turn_bases(T, DIM, 0, [Fraction(8)] * 3, (6, 10) * 3, [90], EXT)
    np.testing.assert_array_equal(b90[:3, :3], [[1, 0, 0], [0, 0, 1], [0, -1, 0]])      # R^T of +90 degrees about +x


def test_a_turn_that_does_not_fit_is_reported():
    occ, labels = _grid()
    _put(occ, labels, np.s_[0], 3)
    _put(occ, labels, np.s_[5, 1:16, 1:16], 1)                          # a 15 x 15 plate: its diagonal is longer than the grid
    axis, _ = PO.down_axis(T, EXT, UP_I)
    _, box, centre = _extent(occ, labels, 1)
    got = OB.turn_bases(T, DIM, axis, centre, box, [0, 45, 90, 135, 180], EXT)
    assert [a for a, bs in got if bs is None] == [45.0, 135.0]
    assert TO.turn_base(T, EXT, DIM, axis, centre, box, 45) is None
    m, _ = _turned(occ, labels, 1, 90.0)
    assert m["drop"].shape == (3, 3) and (m["drop"] == 4).all()
    _put(occ, labels, np.s_[5, 1:16, 1:3], 0, 0.0)                       # a 15 x 13 plate off the middle: the pivot moves
    _, box, centre = _extent(occ, labels, 1)
    assert box == (5, 5, 1, 15, 3, 15) and centre[2] == Fraction(9)
    assert all(bs is not None for _, bs in OB.turn_bases(T, DIM, axis, centre, box, [0, 90, 180, 270], EXT))


def _fake_map(drop, support, offset_lo, centre, lift=0):
    """A placement_map result on the CPU with the keys placement_candidates reads (down -e_i)."""
    return {"drop": torch.tensor(drop), "support": torch.tensor(support), "offset_lo": offset_lo, "axis": 0, "sign": -1,
            "horizontal": [1, 2], "centre": [Fraction(x) for x in centre], "lift": lift, "dim": DIM,
            "_call": (None, None, T, EXT, 0.45, None, None)}


def test_candidates_are_ordered_by_distance_then_turn_then_offset():
    A, b = OB.grid_affine(T, DIM, EXT)
    near = A @ np.array([0.0, 8.0, 8.0]) + b
    m0 = _fake_map([[0, 0, 0], [0, -1, 0], [0, 0, 0]], [[2, 2, -1], [2, -1, 2], [2, 2, 2]], (-1, -1), (4, 9, 9))
    m1 = _fake_map([[1, 0], [0, 0]], [[3, 3], [3, 3]], (-1, -1), (4, 8, 8))
    rows = OB.placement_candidates([m0, m1], near)
    assert rows.shape == (7 + 4, 4)
    assert (np.diff(rows[:, 0]) >= 0).all()
    # distance 0: m0 at (-1, -1) (centre 8, 8) and m1 at (0, 0); the turn order breaks the tie
    np.testing.assert_array_equal(rows[:2, 1:], [[0, -1, -1], [1, 0, 0]])
    ties = rows[np.isclose(rows[:, 0], 0.25 * 1.0)]
    assert [tuple(r[1:]) for r in ties] == sorted(tuple(r[1:]) for r in ties)          # equal distances: turn, then (u, v)
    assert OB.placement_candidates([m0, m1], near, on=[3]).shape[0] == 4
    assert OB.placement_candidates([m0], near, on=[7]).shape == (0, 4)


def test_python_layer_rejects_bad_turn_arguments():
    occ = torch.zeros((DIM,) * 3)
    lab = torch.zeros((DIM,) * 3, dtype=torch.int16)
    eye = np.eye(4)
    args = dict(label=1, down=(0, -1, 0))
    flip = np.diag([1.0, 1.0, -1.0, 1.0])
    row = np.eye(4)
    row[3, 0] = 1.0
    for kw, msg in ((dict(base=np.full((4, 4), np.nan)), "finite"), (dict(base=np.eye(3)), "finite 4x4"),
                    (dict(base=flip), "determinant"), (dict(base=row), "last row"), (dict(box=(0, 1) * 3), "box needs a base"),
                    (dict(base=eye, box=(3, 2, 0, 1, 0, 1)), "inverted"), (dict(base=eye, box=(0, DIM) * 3), "outside the grid"),
                    (dict(base=eye, box=(0, 1)), r"\[1, 6\]")):
        with pytest.raises(ValueError, match=msg):
            OB.placement_map(occ, lab, eye, **dict(args, **kw))
    for turns in (0, -3, True, [], [np.inf], ["x"], "abc", 2.5):
        with pytest.raises(ValueError, match="turns"):
            OB.place_object(occ, lab, eye, near=(0, 0, 0), turns=turns, **args)
    with pytest.raises(RuntimeError, match="CUDA"):
        OB.place_object(occ, lab, eye, near=(0, 0, 0), turns=4, **args)
    assert OB._turn_angles(4) == [0.0, 90.0, 180.0, 270.0] and OB._turn_angles([10, -5.5]) == [10.0, -5.5]


def test_move_objects_and_find_objects_check_the_turns_flag():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import find_objects
    import move_objects
    base = ["ck.tar", "--pose", "p.npy", "--hwk", "4", "4"] + ["1", "0", "2", "0", "1", "2", "0", "0", "1"] + \
        ["--move-label", "1", "--transform", "T.npy", "--out", "o"]
    place = ["--place-at", "0", "1", "2", "--down", "0", "-1", "0"]
    assert move_objects.parse(base + place + ["--turns", "8"]).turns == 8
    assert move_objects.parse(base + place).turns == 1
    assert move_objects.parse(base + place + ["--turns", "1"]).turns == 1
    for extra in (["--mode", "translation", "--turns", "4"], place + ["--turns", "0"], place + ["--turns", "-2"]):
        with pytest.raises(SystemExit):
            move_objects.parse(base + extra)
    fb = ["ck.tar", "--transform", "T.npy", "--out", "d"]
    a = find_objects.parse(fb + ["--placements", "3", "--down", "0", "-1", "0", "--turns", "4"])
    assert a.turns == 4
    assert find_objects.parse(fb + ["--placements", "3", "--down", "0", "-1", "0"]).turns == 1
    for extra in (["--turns", "4"], ["--placements", "3", "--down", "0", "-1", "0", "--turns", "0"]):
        with pytest.raises(SystemExit):
            find_objects.parse(fb + extra)
