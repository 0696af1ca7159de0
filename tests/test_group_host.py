"""CPU: moving objects together -- the numpy restatement (oracle/group_oracle.py) on a hand-built room: a table standing on a
floor with a cup on it and a book on the cup, a shelf and a wall that touches the table top from above.  carried_labels' closure,
the group move landing every member with its layout, the collision checks and placement of the group, a copied group and a
group with a piece, the solid-set equivalence with the same moves one label at a time, the rejections of the Python layer and
the tool, and the ctypes mirror of the group entry points (no GPU)."""
import os
import sys
from fractions import Fraction

import numpy as np
import pytest
import torch

from dmnerf_b200 import _lib
from dmnerf_b200 import objects as OB
from oracle import arrange_oracle as AO
from oracle import collide_oracle as CO
from oracle import edit_sweep_oracle as E
from oracle import group_oracle as GO
from oracle import placement_oracle as PO
from oracle import region_oracle as RO

EXT = (4.0, 4.0, 4.0)
DIM = 17                                             # grid points and 0.25 steps are exact in fp32
T = np.eye(4)
DOWN = (-1.0, 0.0, 0.0)                              # network -x = -e_i: height = index i
LEVEL = 0.45
TABLE, CUP, BOOK, SHELF, WALL, FLOOR = 1, 2, 3, 4, 5, 6
FULL = (0, DIM - 1) * 3


def room():
    """The floor (i 0), a table (top at i 4 over j, k 4..8 on four legs), a cup (i 5..6) on it, a book (i 7) on the cup, a shelf
    board hanging at i 6 beside the table and a wall resting on the table top's edge (j 8)."""
    occ, labels = np.zeros((DIM,) * 3, dtype=np.float32), np.zeros((DIM,) * 3, dtype=np.int16)

    def put(box, label):
        occ[box], labels[box] = 0.9, label
    put(np.s_[0], FLOOR)
    put(np.s_[4, 4:9, 4:9], TABLE)
    for j in (4, 8):
        for k in (4, 8):
            put(np.s_[1:4, j, k], TABLE)
    put(np.s_[5:7, 5:7, 5:7], CUP)
    put(np.s_[7, 5:7, 5:7], BOOK)
    put(np.s_[6, 5:7, 11:13], SHELF)
    put(np.s_[5:12, 8, 4:9], WALL)
    return occ, labels


def _translate(d):
    A, _ = AO.grid_affine(T, DIM, EXT)
    m = np.eye(4)
    m[:3, 3] = -(A @ np.asarray(d, dtype=np.float64))
    return m


def _solid(occ, labels, label):
    return (labels == label) & (occ > np.float32(LEVEL))


def _shifted(mask, d):
    out = np.zeros_like(mask)
    idx = np.argwhere(mask) + np.asarray(d)
    ok = np.all((idx >= 0) & (idx < DIM), axis=1)
    out[tuple(idx[ok].T)] = True
    return out


def _group_box(occ, labels, ks, margin=2):
    mask = np.isin(labels, ks) & (occ > np.float32(LEVEL))
    idx = np.argwhere(mask)
    return tuple(int(x) for a in range(3) for x in (max(idx[:, a].min() - margin, 0), min(idx[:, a].max() + margin, DIM - 1)))


def _gmv(d, occ, labels, group=(TABLE, CUP, BOOK), **kw):
    return dict({"label": group[0], "group": list(group), "trans": _translate(d), "box": _group_box(occ, labels, list(group)),
                 "rest_drop": False}, **kw)


def _grid_edit(occ, labels, moves):
    return GO.grid_edit(occ, labels, occ, labels, T, EXT, moves, LEVEL)


def _centre(occ, labels, label):
    A, b = AO.grid_affine(T, DIM, EXT)
    return A @ np.argwhere(_solid(occ, labels, label)).mean(0) + b


# ---- carried_labels --------------------------------------------------------------------------------------------------------------

def _supports(occ, labels, min_faces=1):
    return OB.supports(OB.contacts_from_faces(CO.object_contacts(occ, labels, LEVEL), T, DIM, EXT), DOWN, min_faces)


def test_carried_labels_finds_cup_and_book_transitively_and_leaves_out_the_floor_and_an_excluded_wall():
    occ, labels = room()
    on = _supports(occ, labels)
    got = OB._carried(on, TABLE, {WALL})
    assert sorted(got["group"]) == [TABLE, CUP, BOOK]
    assert got["chain"][CUP][0] == TABLE and got["chain"][BOOK][0] == CUP and got["chain"][CUP][1] == 4
    assert WALL in OB._carried(on, TABLE, set())["group"]        # the voxelised wall touches the table top from above
    assert FLOOR not in OB._carried(on, TABLE, set())["group"]   # the table rests on the floor, not the other way round
    assert OB._carried(on, CUP, set())["group"] == [CUP, BOOK]
    assert OB._carried(_supports(occ, labels, min_faces=5), TABLE, {WALL})["group"] == [TABLE]   # the cup touches 4 faces


# ---- the grid edit --------------------------------------------------------------------------------------------------------------

def test_the_group_move_lands_all_three_with_their_layout_and_centres_move_together():
    occ, labels = room()
    d = (0, 0, 6)
    o, l, landed, over = _grid_edit(occ, labels, [_gmv(d, occ, labels)])
    A, _ = AO.grid_affine(T, DIM, EXT)
    for k in (TABLE, CUP, BOOK):
        assert np.array_equal(_solid(o, l, k), _shifted(_solid(occ, labels, k), d)), k
        np.testing.assert_allclose(_centre(o, l, k) - _centre(occ, labels, k), A @ np.asarray(d, dtype=np.float64), rtol=0,
                                   atol=1e-12)
    assert landed[0] == sum(_solid(occ, labels, k).sum() for k in (TABLE, CUP, BOOK))
    assert over[0][SHELF] == 4 and over[0][[TABLE, CUP, BOOK]].sum() == 0   # only the cup lands on the shelf
    for k in (FLOOR, WALL):
        assert np.array_equal(_solid(o, l, k), _solid(occ, labels, k))


def test_a_group_of_one_is_the_single_move_and_absent_or_identity_groups_change_nothing():
    occ, labels = room()
    single = {"label": CUP, "trans": _translate((0, 3, 0)), "box": FULL, "rest_drop": False}
    a = _grid_edit(occ, labels, [single])
    b = _grid_edit(occ, labels, [dict(single, group=[CUP])])
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    for mv in (dict(single, label=9, group=[9, 10]), _gmv((0, 0, 0), occ, labels)):
        o, l, _, _ = _grid_edit(occ, labels, [mv])
        assert np.array_equal(o, occ) and np.array_equal(l, labels)


def test_a_copied_group_keeps_its_source_and_a_piece_cuts_only_the_labels_it_applies_to():
    occ, labels = room()
    d = (0, 0, 8)
    o, l, _, _ = _grid_edit(occ, labels, [_gmv(d, occ, labels, copy=True)])
    for k in (TABLE, CUP, BOOK):
        src = _solid(occ, labels, k)
        assert np.array_equal(_solid(o, l, k), src | _shifted(src, d)), k
    half = np.zeros((DIM,) * 3, dtype=bool)
    half[:, :, :6] = True                              # k <= 5: two columns of the table top, half of the cup
    A, b = OB.grid_affine(T, DIM, EXT)
    piece = E.Piece(RO.pack(half), DIM, RO.voxel_map(A, b), outside_keep=True)
    o, l, _, _ = _grid_edit(occ, labels, [_gmv(d, occ, labels, piece=piece, applies=[TABLE])])
    table = _solid(occ, labels, TABLE)
    assert np.array_equal(_solid(o, l, TABLE), (table & ~half) | _shifted(table & half, d))
    for k in (CUP, BOOK):                              # the piece does not apply to them: they move whole
        assert np.array_equal(_solid(o, l, k), _shifted(_solid(occ, labels, k), d)), k


def test_the_group_equals_its_moves_one_label_at_a_time_on_solid_points():
    rng = np.random.default_rng(11)
    occ = rng.uniform(0.0, 1.0, (DIM,) * 3).astype(np.float32)
    labels = rng.integers(0, 4, (DIM,) * 3).astype(np.int16)
    inv, b = E.grid_index_map(T, EXT, DIM)
    ev = E.grid_evaluate(occ, labels.astype(np.int64), inv, b)
    lev = np.float32(LEVEL)
    for (la, lb), trans in (((1, 2), _translate((0, 2, -1))), ((3, 0), _translate((1, 0, 1))), ((2, 1), _translate((0, 0, 0)))):
        group = {"label": la, "group": [la, lb], "trans": trans, "box": FULL}
        seq = [{"label": la, "trans": trans, "box": FULL}, {"label": lb, "trans": trans, "box": FULL}]
        for run in (lambda ms: GO.edit(occ, labels, T, EXT, ms, ev, LEVEL)[:2], lambda ms: _grid_edit(occ, labels, ms)[:2]):
            go, gl = run([group])
            so, sl = run(seq)
            solid = go > lev
            assert np.array_equal(solid, so > lev)
            np.testing.assert_array_equal(go[solid], so[solid])
            np.testing.assert_array_equal(gl[solid], sl[solid])
            # below the level: only air the sequence takes with label B where the group vacates
            diff = (go != so) | (gl != sl)
            assert (go[diff] == 0).all() and (gl[diff] == la).all() and (sl[diff] == lb).all() and (so[diff] <= lev).all()


# ---- collision checks and placement ----------------------------------------------------------------------------------------------

def test_move_overlap_of_the_group_reports_the_shelf_the_cup_hits_and_no_overlap_inside_the_group():
    occ, labels = room()
    over, landed = GO.move_overlap(occ, labels, T, EXT, [_gmv((0, 0, 6), occ, labels)], LEVEL)
    assert over[0][SHELF] == 4 and over[0].sum() == 4
    over, _ = GO.move_overlap(occ, labels, T, EXT, [_gmv((1, 0, 0), occ, labels)], LEVEL)    # raised by one voxel
    assert over[0][[TABLE, CUP, BOOK]].sum() == 0
    table = {"label": TABLE, "trans": _translate((1, 0, 0)), "box": _group_box(occ, labels, [TABLE])}
    alone, _ = CO.move_overlap(occ, labels, T, EXT, [table], LEVEL)
    assert alone[0][CUP] > 0                           # the table raised alone runs into its own cup
    over, _ = GO.move_overlap(occ, labels, T, EXT, [_gmv((1, 0, 0), occ, labels, copy=True)], LEVEL)
    assert over[0][TABLE] > 0                          # a copied group: the source stays an obstacle


def test_the_group_rests_on_the_floor_never_on_a_member_and_its_stability_uses_the_group_centre():
    occ, labels = room()
    axis, sign = PO.down_axis(T, EXT, DOWN)
    mv = _gmv((0, 0, 0), occ, labels)
    m = GO.placement_in_scene(occ, labels, occ, labels, T, EXT, mv, LEVEL, axis, sign, 0)
    u0, v0 = m["offset_lo"]
    assert m["drop"][-u0, -v0] == 0 and m["support"][-u0, -v0] == FLOOR
    members = np.isin(labels, [TABLE, CUP, BOOK]) & (occ > np.float32(LEVEL))
    assert m["points"].shape[0] == members.sum()
    pts = np.argwhere(PO.to_columns(members, axis, sign))
    assert m["centre"] == [Fraction(int(s), pts.shape[0]) for s in pts.sum(0)]   # the cup and book count towards the centre
    supported = m["support"][m["support"] >= 0]
    assert not np.isin(supported, [TABLE, CUP, BOOK]).any()
    assert PO.stable(m, -u0, -v0)
    cup = GO.placement_in_scene(occ, labels, occ, labels, T, EXT, _gmv((0, 0, 0), occ, labels, group=(CUP, BOOK)), LEVEL, axis,
                                sign, 0)
    assert cup["support"][-cup["offset_lo"][0], -cup["offset_lo"][1]] == TABLE   # the cup and book rest on the table


# ---- the Python layer's checks ----------------------------------------------------------------------------------------------------

def test_groups_parse_and_check_their_labels():
    assert OB.move_groups(None, [1, 2], 13) is None
    assert OB.move_groups([None, None], [1, 2], 13) is None
    assert OB.move_groups([[3, 1, 3], None], [1, 2], 13) == [(1, 3), (2,)]
    assert OB.move_groups(((1, 2),), [1], 13) == [(1, 2)]
    for bad, msg in (([[2]], "does not hold"), ([[1, 14]], "outside"), ([[1, 2]] * 2, "one entry per move"), ([3], "iterable"),
                     ("12", "groups must be"), ([[1.5]], "integers")):
        with pytest.raises(ValueError, match=msg):
            OB.move_groups(bad, [1], 13)


def test_the_order_rule_is_per_label_of_the_sets():
    sets = [(1, 2), (2, 3)]
    with pytest.raises(ValueError, match="move 1 of label 2 follows copy 0"):
        OB._check_copies([True, False], [1, 3], [False, False], sets=sets)
    assert OB._check_copies([True, False], [1, 3], [False, False], sets=[(1, 2), (3,)]) == [True, False]
    assert OB._check_copies([False, True], [1, 3], [False, False], sets=sets) == [False, True]
    assert OB._check_copies([True, False], [1, 3], [False, False], ordered=False, sets=sets) == [True, False]


def test_python_layer_rejects_bad_groups_before_any_device_work():
    occ, labels = torch.zeros((DIM,) * 3), torch.zeros((DIM,) * 3, dtype=torch.int16)
    m = [(TABLE, np.eye(4))]
    calls = [
        (lambda: OB.render_moves(occ, labels, T, m, EXT, groups=[[CUP]]), "does not hold"),
        (lambda: OB.render_moves(occ, labels, T, m, EXT, groups=[[TABLE, 200]]), "outside"),
        (lambda: OB.render_moves(occ, labels, T, m * 2, EXT, copies=[True, False], groups=[[TABLE, CUP], None]), "follows copy"),
        (lambda: OB.edit_boxes(occ, labels, m, T, EXT, groups=[[TABLE], [CUP]]), "one entry per move"),
        (lambda: OB.placement_map(occ, labels, T, TABLE, DOWN, extents=EXT, group=[CUP]), "does not hold"),
        (lambda: OB.place_object(occ, labels, T, TABLE, DOWN, (0, 0, 0), on=[CUP], extents=EXT, group=[TABLE, CUP]),
         "never rests on itself"),
        (lambda: OB.turned_placement_maps(occ, labels, T, TABLE, DOWN, 4, extents=EXT, group=[TABLE, 300]), "outside"),
    ]
    for call, msg in calls:
        with pytest.raises(ValueError, match=msg):
            call()
    with pytest.raises(RuntimeError, match="CUDA"):    # a good group passes the checks and then needs the device
        OB.render_moves(occ, labels, T, m, EXT, groups=[[TABLE, CUP]])


def test_arrange_items_take_a_group_and_reject_move_items_whose_sets_intersect():
    occ, labels = torch.zeros((DIM,) * 3), torch.zeros((DIM,) * 3, dtype=torch.int16)
    table = {"label": TABLE, "near": (0.0, 0.0, 0.0), "group": [TABLE, CUP]}
    cup = {"label": CUP, "near": (0.0, 0.0, 0.0)}
    for items, msg in (([table, cup], "share label 2"), ([dict(cup, copy=True), table], "moves label 2 after item 0 copies it"),
                       ([dict(table, group=[CUP])], "does not hold"), ([dict(table, on=[CUP])], "never rests on itself")):
        with pytest.raises(ValueError, match=msg):
            OB.arrange_objects(occ, labels, T, items, DOWN, EXT)
    for items in ([table, dict(cup, copy=True)], [table, {"label": BOOK, "near": (0.0, 0.0, 0.0)}]):
        with pytest.raises(RuntimeError, match="CUDA"):
            OB.arrange_objects(occ, labels, T, items, DOWN, EXT)


def test_moved_scene_defaults_to_each_moves_own_label():
    d = _lib.RenderMoves()
    ms = OB.MovedScene(d, (), torch.device("cpu"), (1, 2), np.zeros((2, 6), dtype=np.int64), [False, False], 0.45, 0.1)
    assert ms.groups == ((1,), (2,)) and ms.group_words() is None
    ms = OB.MovedScene(d, (), torch.device("cpu"), (1, 2), np.zeros((2, 6), dtype=np.int64), [False, False], 0.45, 0.1, None,
                       [(1, 3), (2,)])
    assert ms.groups == ((1, 3), (2,)) and list(ms.group_words()) == [0b1010, 0, 0, 0, 0b100, 0, 0, 0]


# ---- the C ABI and the tool -----------------------------------------------------------------------------------------------------

def test_group_entry_points_are_the_copy_ones_with_a_label_set_argument():
    P = _lib.PROTOTYPES
    words = _lib.C.POINTER(_lib.C.c_uint32)
    for name, at in (("dmnerf_mesh_occupancy_edit", 10), ("dmnerf_grid_edit", 9), ("dmnerf_render_moved", 9),
                     ("dmnerf_move_overlap", 9)):
        base, new = P[name + "_copies"], P[name + "_groups"]
        assert new[0] is base[0] and new[1][at] is words and new[1][:at] + new[1][at + 1:] == base[1], name
    for name in ("dmnerf_placement_maps_in_scene", "dmnerf_placement_contacts_in_scene"):
        base, new = P[name + "_copy"], P[name + "_group"]
        assert new[1][11] is words and new[1][:11] + new[1][12:] == base[1], name


def test_the_tool_takes_with_and_carry_and_needs_the_per_sample_render(tmp_path, capsys):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import move_objects
    base = ["ck.tar", "--pose", "p.npy", "--hwk", "4", "4"] + ["1"] * 9 + ["--transform", "t.npy", "--out", "o"]
    mv = ["--move-label", "1", "--mode", "translation", "--render", "samples"]
    a = move_objects.parse(base + mv + ["--with", "2", "3"])
    assert a.with_labels == [2, 3] and a.grouped
    assert move_objects.parse(base + mv + ["--carry", "--down", "0", "-1", "0"]).carry
    assert move_objects.parse(base + ["--move-label", "1", "--place-at", "0", "0", "0", "--down", "0", "-1", "0", "--carry",
                                      "--render", "samples"]).carry
    assert move_objects.parse(base + mv + ["--with", "2", "--check"]).check
    spec = tmp_path / "spec.json"
    spec.write_text('[{"label": 1, "near": [0, 0, 0], "group": [1, 2]}]')
    assert move_objects.read_spec(str(spec))[0]["group"] == [1, 2]
    for extra, msg in ((["--move-label", "1", "--mode", "translation", "--with", "2"], "--render samples"),
                       (mv + ["--carry"], "--carry needs --down"),
                       (mv + ["--with", "2", "--until-contact"], "until-contact"),
                       (["--arrange", str(spec), "--down", "0", "-1", "0", "--with", "2", "--render", "samples"], "per item")):
        with pytest.raises(SystemExit):
            move_objects.parse(base + extra)
        assert msg in capsys.readouterr().err, msg
    for text, msg in (('[{"label": 1, "near": [0, 0, 0], "group": 2}]', "group must be a list of labels"),
                      ('[{"label": 1, "near": [0, 0, 0], "group": [2, 3]}]', "does not hold the item's label 1")):
        spec.write_text(text)
        with pytest.raises(SystemExit, match=msg):
            move_objects.read_spec(str(spec))
