"""CPU: copying objects -- the numpy restatement (oracle/copy_oracle.py) on hand-built grids: one and several copies of a label, a
copy after a move of its label, a copy landing on its source, a piece copied, the source as an obstacle of move_overlap, a box
stacked on its own copy, four copies of a chair around a table; the rejections of the Python layer; and the ctypes mirror of the
copy entry points (no GPU)."""
import numpy as np
import pytest
import torch

from dmnerf_b200 import _lib
from dmnerf_b200 import objects as OB
from oracle import arrange_oracle as AO
from oracle import collide_oracle as CO
from oracle import copy_oracle as CP
from oracle import edit_sweep_oracle as E
from oracle import region_oracle as RO

EXT = (4.0, 4.0, 4.0)
DIM = 17                                             # grid points and 0.25 steps are exact in fp32
T = np.eye(4)
DOWN = (-1.0, 0.0, 0.0)                              # network -x = -e_i: height = index i
LEVEL = 0.45
FLOOR, TABLE, BOX, CHAIR = 6, 1, 2, 3


def _grid():
    occ, labels = np.zeros((DIM,) * 3, dtype=np.float32), np.zeros((DIM,) * 3, dtype=np.int16)
    occ[0], labels[0] = 0.9, FLOOR
    return occ, labels


def _put(occ, labels, box, label, value=0.9):
    occ[box], labels[box] = value, label


def _net(i, j, k):
    A, b = AO.grid_affine(T, DIM, EXT)
    return A @ np.array([i, j, k], dtype=np.float64) + b


def _translate(d):
    """The move that lands an object at x + A d (index displacement d)."""
    A, _ = AO.grid_affine(T, DIM, EXT)
    m = np.eye(4)
    m[:3, 3] = -(A @ np.asarray(d, dtype=np.float64))
    return m


def _solid(occ, labels, label):
    return (labels == label) & (occ > np.float32(LEVEL))


def _mv(label, d, occ, labels, copy=True, piece=None, trans=None):
    return {"label": label, "trans": _translate(d) if trans is None else trans, "piece": piece, "rest_drop": False, "copy": copy,
            "box": E.solid_box(occ, labels, label, LEVEL, 2)}


def _shifted(mask, d):
    out = np.zeros_like(mask)
    idx = np.argwhere(mask) + np.asarray(d)
    ok = np.all((idx >= 0) & (idx < DIM), axis=1)
    out[tuple(idx[ok].T)] = True
    return out


def _box_scene():
    occ, labels = _grid()
    _put(occ, labels, np.s_[1:3, 3:5, 3:5], BOX)
    return occ, labels


def _grid_edit(occ, labels, moves):
    return CP.grid_edit(occ, labels, occ, labels, T, EXT, moves, LEVEL)


# ---- the grid edit --------------------------------------------------------------------------------------------------------------

def test_one_copy_keeps_the_source_and_lands_a_second_piece_of_the_label():
    occ, labels = _box_scene()
    src = _solid(occ, labels, BOX)
    o, l, landed, over = _grid_edit(occ, labels, [_mv(BOX, (0, 6, 6), occ, labels)])
    assert np.array_equal(_solid(o, l, BOX), src | _shifted(src, (0, 6, 6)))
    assert landed[0] == src.sum() and over[0].sum() == 0
    move_o, move_l, _, _ = _grid_edit(occ, labels, [_mv(BOX, (0, 6, 6), occ, labels, copy=False)])
    assert np.array_equal(_solid(move_o, move_l, BOX), _shifted(src, (0, 6, 6)))


def test_several_copies_of_one_label_each_land_and_the_source_stays():
    occ, labels = _box_scene()
    src = _solid(occ, labels, BOX)
    ds = [(0, 6, 0), (0, 0, 6), (0, 6, 6), (2, 0, 0)]
    o, l, landed, _ = _grid_edit(occ, labels, [_mv(BOX, d, occ, labels) for d in ds])
    want = src.copy()
    for d in ds:
        want |= _shifted(src, d)
    assert np.array_equal(_solid(o, l, BOX), want) and (landed == src.sum()).all()


def test_a_copy_after_a_move_of_its_label_copies_the_unedited_object():
    occ, labels = _box_scene()
    src = _solid(occ, labels, BOX)
    o, l, _, _ = _grid_edit(occ, labels, [_mv(BOX, (0, 8, 0), occ, labels, copy=False), _mv(BOX, (0, 0, 8), occ, labels)])
    assert np.array_equal(_solid(o, l, BOX), _shifted(src, (0, 8, 0)) | _shifted(src, (0, 0, 8)))


def test_a_copy_landing_on_its_source_counts_its_own_points_and_an_identity_copy_changes_nothing():
    occ, labels = _box_scene()
    src = _solid(occ, labels, BOX)
    o, l, landed, over = _grid_edit(occ, labels, [_mv(BOX, (0, 0, 0), occ, labels)])
    assert np.array_equal(o, occ) and np.array_equal(l, labels)
    assert over[0][BOX] == src.sum()                     # a copy vacates nothing: it lands on its own source
    o, l, _, over = _grid_edit(occ, labels, [_mv(BOX, (0, 1, 0), occ, labels)])
    assert np.array_equal(_solid(o, l, BOX), src | _shifted(src, (0, 1, 0)))
    assert over[0][BOX] == (src & _shifted(src, (0, 1, 0))).sum()
    _, _, _, over_move = _grid_edit(occ, labels, [_mv(BOX, (0, 1, 0), occ, labels, copy=False)])
    assert over_move[0][BOX] == 0


def test_an_absent_label_or_the_empty_box_changes_nothing():
    occ, labels = _box_scene()
    for mv in ({"label": 9, "trans": _translate((0, 3, 0)), "box": (0, DIM - 1) * 3, "copy": True},
               {"label": BOX, "trans": _translate((0, 3, 0)), "box": E.EMPTY_BOX, "copy": True}):
        o, l, landed, over = _grid_edit(occ, labels, [mv])
        assert np.array_equal(o, occ) and np.array_equal(l, labels) and landed[0] == 0 and over.sum() == 0


def test_copy_equals_the_move_where_the_move_takes_and_the_input_elsewhere():
    rng = np.random.default_rng(7)
    occ = rng.uniform(0.0, 1.0, (DIM,) * 3).astype(np.float32)
    labels = rng.integers(0, 4, (DIM,) * 3).astype(np.int16)
    inv, b = E.grid_index_map(T, EXT, DIM)
    ev = E.grid_evaluate(occ, labels.astype(np.int64), inv, b)
    for label, d in ((1, (0, 2, -1)), (2, (1, 0, 0))):
        mv = _mv(label, d, occ, labels, copy=False)
        take, _, _ = CP.take_mask(occ.reshape(-1), E.sweep_points(T, EXT, DIM), inv, b, mv, ev, LEVEL)
        take = take.reshape(occ.shape)
        move_o, move_l, _ = E.edit(occ, labels, T, EXT, [mv], ev, LEVEL)
        copy_o, copy_l, _ = CP.edit(occ, labels, T, EXT, [dict(mv, copy=True)], ev, LEVEL)
        assert take.any()
        np.testing.assert_array_equal(copy_o[take], move_o[take])
        np.testing.assert_array_equal(copy_l[take], move_l[take])
        np.testing.assert_array_equal(copy_o[~take], occ[~take])
        np.testing.assert_array_equal(copy_l[~take], labels[~take])
        go, gl, _, _ = _grid_edit(occ, labels, [dict(mv, copy=True)])
        np.testing.assert_array_equal(go, copy_o)
        np.testing.assert_array_equal(gl, copy_l)


def _piece(mask):
    A, b = OB.grid_affine(np.eye(4), DIM, EXT)
    return E.Piece(RO.pack(mask), DIM, RO.voxel_map(A, b), outside_keep=True)


def test_a_piece_copied_leaves_the_whole_label_and_lands_only_the_piece():
    occ, labels = _grid()
    _put(occ, labels, np.s_[1:3, 3:9, 3:5], BOX)
    src = _solid(occ, labels, BOX)
    half = np.zeros_like(src)
    half[:, 3:6] = True
    mv = {"label": BOX, "trans": _translate((0, 0, 8)), "box": (0, DIM - 1) * 3, "piece": _piece(half), "copy": True}
    o, l, landed, _ = _grid_edit(occ, labels, [mv])
    assert np.array_equal(_solid(o, l, BOX), src | _shifted(src & half, (0, 0, 8)))
    assert landed[0] == (src & half).sum()


# ---- collision checks and placement -----------------------------------------------------------------------------------------------

def test_move_overlap_of_a_copy_counts_its_source_as_an_obstacle():
    occ, labels = _box_scene()
    src = _solid(occ, labels, BOX)
    for d in ((0, 0, 0), (0, 1, 0), (0, 1, 1)):
        mv = _mv(BOX, d, occ, labels)
        over, landed = CP.move_overlap(occ, labels, T, EXT, [mv], LEVEL)
        assert landed[0] == src.sum() and over[0][BOX] == (src & _shifted(src, d)).sum()
        m_over, m_landed = CO.move_overlap(occ, labels, T, EXT, [dict(mv, copy=False)], LEVEL)
        assert m_landed[0] == landed[0] and m_over[0][BOX] == 0
    over, _ = CP.move_overlap(occ, labels, T, EXT, [_mv(BOX, (0, 1, 0), occ, labels)], LEVEL, obstacles=[FLOOR])
    assert over[0].sum() == 0


def test_a_box_stacks_on_its_own_copy():
    occ, labels = _box_scene()
    items = [{"label": BOX, "near": _net(0, 4, 4), "on": [BOX], "copy": True, "lift": 2}]   # raised clear of its source
    o, l, chosen = CP.arrange(occ, labels, T, EXT, items, DOWN, LEVEL)
    src = _solid(occ, labels, BOX)
    assert chosen[0] is not None and chosen[0]["offset"] == (0, 0) and chosen[0]["drop"] == 0
    assert np.array_equal(_solid(o, l, BOX), src | _shifted(src, (2, 0, 0)))     # the copy sits on top of its source
    items = [{"label": BOX, "near": _net(0, 4, 4), "on": [BOX], "lift": 2}]       # a move vacates its source: nothing to rest on
    _, _, moved = CP.arrange(occ, labels, T, EXT, items, DOWN, LEVEL)
    assert moved[0] is None


def _chair_scene():
    """A floor, a table (label 1: a top at i 4 on four legs) in the middle and a chair (label 3) in a corner."""
    occ, labels = _grid()
    _put(occ, labels, np.s_[4, 6:11, 6:11], TABLE)
    for j in (6, 10):
        for k in (6, 10):
            _put(occ, labels, np.s_[1:4, j, k], TABLE)
    _put(occ, labels, np.s_[1:3, 1:3, 1:3], CHAIR)
    _put(occ, labels, np.s_[3:5, 1, 1:3], CHAIR)
    return occ, labels


def test_four_copies_of_a_chair_arranged_around_a_table():
    occ, labels = _chair_scene()
    spots = [(0, 8, 3), (0, 8, 13), (0, 3, 8), (0, 13, 8)]
    items = [{"label": CHAIR, "near": _net(*s), "on": [FLOOR], "copy": True} for s in spots]
    o, l, chosen = CP.arrange(occ, labels, T, EXT, items, DOWN, LEVEL)
    assert all(c is not None for c in chosen)
    chair = _solid(occ, labels, CHAIR)
    assert _solid(o, l, CHAIR).sum() == 5 * chair.sum()                          # the source and four copies, apart
    assert np.array_equal(_solid(o, l, TABLE), _solid(occ, labels, TABLE))
    for c in chosen:
        u, v = c["offset"]
        assert c["drop"] == 0 and (u, v) != (0, 0)


# ---- the Python layer's checks ----------------------------------------------------------------------------------------------------

def test_copy_flags_parse_like_rest():
    assert OB.move_copies(None, 2) == [False, False]
    assert OB.move_copies(True, 3) == [True, True, True]
    assert OB.move_copies([True, False], 2) == [True, False]
    assert OB.move_copies(np.array([True, False]), 2) == [True, False]
    for bad in ([True], [1, 0], 1, [2, 0], "yes", 0.5, [None, True]):
        with pytest.raises(ValueError, match="copies"):
            OB.move_copies(bad, 2)


def test_python_layer_rejects_bad_copies_before_any_device_work():
    occ, labels = torch.zeros((DIM,) * 3), torch.zeros((DIM,) * 3, dtype=torch.int16)
    m = [(BOX, np.eye(4))]
    calls = [
        (lambda: OB.render_moves(occ, labels, T, m * 2, EXT, copies=[True, 2]), "copies"),
        (lambda: OB.render_moves(occ, labels, T, m * 2, EXT, copies=[True, False]), "follows copy"),
        (lambda: OB.render_moves(occ, labels, T, m, EXT, rest="drop", copies=True), "drop"),
        (lambda: OB.placement_map(occ, labels, T, BOX, DOWN, extents=EXT, rest="drop", copy=True), "drop"),
        (lambda: OB.place_object(occ, labels, T, BOX, DOWN, (0, 0, 0), extents=EXT, copy=2), "copies"),
        (lambda: OB.turned_placement_maps(occ, labels, T, BOX, DOWN, 4, extents=EXT, rest="drop", copy=True), "drop"),
    ]
    for call, msg in calls:
        with pytest.raises(ValueError, match=msg):
            call()
    # the shared check of edited_sweep, edited_grid, edit_occupancy, move_overlap and render_moves
    assert OB._check_copies([False, True, True], [BOX] * 3, [False] * 3) == [False, True, True]   # copies after a move
    with pytest.raises(ValueError, match="follows copy 0"):
        OB._check_copies([True, False], [BOX, BOX], [False, False])
    assert OB._check_copies([True, False], [BOX, BOX], [False, False], ordered=False) == [True, False]   # candidates
    assert OB._check_copies([True, False], [BOX, TABLE], [False, False]) == [True, False]
    with pytest.raises(ValueError, match="drop"):
        OB._check_copies(True, [BOX], [True], ordered=False)
    # a copy after a move of its label and several copies of one label pass the checks (and then need the device)
    with pytest.raises(RuntimeError, match="CUDA"):
        OB.render_moves(occ, labels, T, m * 3, EXT, copies=[False, True, True])


def test_arrange_items_take_copy_and_reject_a_move_after_a_copy():
    occ, labels = torch.zeros((DIM,) * 3), torch.zeros((DIM,) * 3, dtype=torch.int16)
    ok = {"label": BOX, "near": (0.0, 0.0, 0.0)}
    cp = dict(ok, copy=True)
    for items, msg in (([ok, dict(ok)], "share label"), ([cp, ok], "after item 0 copies it"), ([dict(cp, rest="drop")], "drop"),
                       ([dict(ok, copy=1)], "copy must be")):
        with pytest.raises(ValueError, match=msg):
            OB.arrange_objects(occ, labels, T, items, DOWN, EXT)
    for items in ([ok, cp], [cp, cp, dict(cp, on=[BOX])]):
        with pytest.raises(RuntimeError, match="CUDA"):             # checked, then the device is needed
            OB.arrange_objects(occ, labels, T, items, DOWN, EXT)


def test_moved_scene_defaults_to_no_copies():
    d = _lib.RenderMoves()
    ms = OB.MovedScene(d, (), torch.device("cpu"), (1, 1), np.zeros((2, 6), dtype=np.int64), [False, False], 0.45, 0.1)
    assert ms.copies == (False, False) and ms.copy_flags() is None
    ms = OB.MovedScene(d, (), torch.device("cpu"), (1, 1), np.zeros((2, 6), dtype=np.int64), [False, False], 0.45, 0.1, [False, True])
    assert ms.copies == (False, True) and list(ms.copy_flags()) == [0, 1]
    with pytest.raises(AttributeError):
        ms.copies = (True, True)


# ---- the C ABI ---------------------------------------------------------------------------------------------------------------------

def test_copy_entry_points_are_their_namesakes_with_a_flag_argument():
    P = _lib.PROTOTYPES
    flags = _lib.C.POINTER(_lib.C.c_int32)
    for name, at in (("dmnerf_mesh_occupancy_edit", 9), ("dmnerf_grid_edit", 8), ("dmnerf_render_moved", 8),
                     ("dmnerf_move_overlap", 8)):
        base, new = P[name], P[name + "_copies"]
        assert new[0] is base[0] and new[1][at] is flags and new[1][:at] + new[1][at + 1:] == base[1], name
    for name in ("dmnerf_placement_maps_in_scene", "dmnerf_placement_contacts_in_scene"):
        base, new = P[name], P[name + "_copy"]
        assert new[1][10] is _lib.C.c_int and new[1][:10] + new[1][11:] == base[1], name


def test_the_tool_takes_copy_per_item_with_arrange_and_needs_the_per_sample_render(tmp_path):
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import move_objects
    spec = tmp_path / "spec.json"
    spec.write_text('[{"label": 1, "near": [0, 0, 0], "copy": true}]')
    base = ["ck.tar", "--pose", "p.npy", "--hwk", "4", "4"] + ["1"] * 9 + ["--transform", "t.npy", "--out", "o"]
    assert move_objects.parse(base + ["--move-label", "1", "--mode", "translation", "--copy", "--render", "samples"]).copy
    assert move_objects.read_spec(str(spec))[0]["copy"] is True
    for extra in (["--move-label", "1", "--mode", "translation", "--copy"],                       # the exchanger moves only
                  ["--move-label", "1", "--mode", "translation", "--copy", "--render", "samples", "--rest", "drop"],
                  ["--move-label", "1", "--mode", "translation", "--copy", "--render", "samples", "--until-contact"],
                  ["--arrange", str(spec), "--down", "0", "-1", "0", "--copy", "--render", "samples"]):   # copy is per item
        with pytest.raises(SystemExit):
            move_objects.parse(base + extra)
    spec.write_text('[{"label": 1, "near": [0, 0, 0], "copy": 1}]')
    with pytest.raises(SystemExit):
        move_objects.read_spec(str(spec))

