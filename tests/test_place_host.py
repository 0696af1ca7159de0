"""CPU: object placement -- the numpy restatement of the rule (oracle/placement_oracle.py) on hand-built grids, the exact hull
test, the transformation's convention against the collision checks, and the argument checks of the Python layer and of the
tools (no GPU)."""
import os
import sys
from fractions import Fraction

import numpy as np
import pytest
import torch

from dmnerf_b200 import objects as OB
from oracle import collide_oracle as CO
from oracle import placement_oracle as PO
from oracle import region_oracle as RO
from oracle import edit_sweep_oracle as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXT = (4.0, 4.0, 4.0)
DIM = 17                                             # grid points and 0.25 steps are exact in fp32
T = np.eye(4)
UP_I = (-1.0, 0.0, 0.0)                              # network -x = -e_i: height = index i


def _grid():
    return np.zeros((DIM,) * 3, dtype=np.float32), np.zeros((DIM,) * 3, dtype=np.int16)


def _put(occ, labels, box, label, value=0.9):
    occ[box], labels[box] = value, label


def _map(occ, labels, label, lift=0, down=UP_I, **kw):
    axis, sign = PO.down_axis(T, EXT, down)
    return PO.placement_map(occ, labels, T, EXT, label, 0.45, axis, sign, lift, **kw)


def _at(m, u, v, key):
    return int(m[key][u - m["offset_lo"][0], v - m["offset_lo"][1]])


def test_down_is_chosen_as_supports_chooses_it():
    A, _ = OB.grid_affine(T, DIM, EXT)
    axes = (A / np.linalg.norm(A, axis=0)).T
    for down in ((-1, 0, 0), (1, 0.2, 0), (0, -1, 0), (0, 1, 0.3), (0, 0, 1), (0.1, 0, -1)):
        assert PO.down_axis(T, EXT, down) == OB.down_axis(axes, down, "t")
    assert PO.down_axis(T, EXT, UP_I) == (0, -1)
    assert PO.down_axis(T, EXT, (0, -1, 0)) == (2, 1)           # network -y is +e_k


def test_a_cube_above_a_slab_drops_exactly_the_gap():
    for gap in (0, 1, 4):
        occ, labels = _grid()
        _put(occ, labels, np.s_[0:2], 3)
        _put(occ, labels, np.s_[2 + gap:5 + gap, 4:7, 4:7], 1)
        m = _map(occ, labels, 1)
        assert m["offset_lo"] == (-4, -4) and m["drop"].shape == (DIM - 2, DIM - 2)
        assert (m["drop"] == gap).all() and (m["contacts"] == 9).all() and (m["support"] == 3).all()
        assert m["centre"] == [Fraction(5), Fraction(5), Fraction(3 + gap)]


def _table():
    """Floor (label 3) at i 0..1; a table (label 2): top at i 8, j, k 3..12, legs at the four corners; a 2^3 box (label 1) on
    the floor beside it at j, k 14..15."""
    occ, labels = _grid()
    _put(occ, labels, np.s_[0:2], 3)
    _put(occ, labels, np.s_[8, 3:13, 3:13], 2)
    for j in (3, 12):
        for k in (3, 12):
            _put(occ, labels, np.s_[2:8, j, k], 2)
    _put(occ, labels, np.s_[2:4, 14:16, 14:16], 1)
    return occ, labels


def test_a_box_beside_a_table_rests_under_it_or_on_it():
    occ, labels = _table()
    m = _map(occ, labels, 1)
    assert m["offset_lo"] == (-14, -14)
    assert _at(m, 0, 0, "drop") == 0 and _at(m, 0, 0, "support") == 3
    assert _at(m, -7, -7, "drop") == 0 and _at(m, -7, -7, "support") == 3          # under the top, between the legs
    assert _at(m, -11, -11, "drop") == -1 and _at(m, -11, -11, "support") == -1    # j, k 3..4: the leg at (3, 3)
    assert _at(m, -11, -11, "contacts") == 0
    blocked = m["drop"] < 0
    assert blocked.sum() == 4 * 4 and ((m["support"] == 3) | blocked).all()             # 4 legs x 4 offsets each (2x2 box)
    m = _map(occ, labels, 1, lift=7)
    assert _at(m, -7, -7, "drop") == 0 and _at(m, -7, -7, "support") == 2 and _at(m, -7, -7, "contacts") == 4
    assert _at(m, 0, 0, "drop") == 7 and _at(m, 0, 0, "support") == 3
    assert _at(m, -2, -2, "drop") == 0 and _at(m, -2, -2, "support") == 2
    assert _at(m, -2, -2, "contacts") == 1                                         # one corner of the box on the top's corner
    assert (m["drop"] >= 0).all()
    m = _map(occ, labels, 1, lift=7, obstacles=[3])                                   # the table is left out
    assert _at(m, -7, -7, "drop") == 7 and _at(m, -7, -7, "support") == 3


def test_runs_interleaved_with_an_obstacle_are_blocked_or_drop_correctly():
    """Label 1 has two runs in one column, at i 3 and i 10, with a shelf (label 4) at i 6..8 between them; floor at i 0..1."""
    occ, labels = _grid()
    _put(occ, labels, np.s_[0:2], 3)
    _put(occ, labels, np.s_[6:9, 7, 6], 4)
    _put(occ, labels, np.s_[3, 7, 6], 1)
    _put(occ, labels, np.s_[10, 7, 6], 1)
    m0 = _map(occ, labels, 1)
    assert _at(m0, 0, 0, "drop") == 1 and _at(m0, 0, 0, "contacts") == 2
    assert _at(m0, 0, 0, "support") == 3                                # one run on the floor, one on the shelf: ties to 3
    for lift, want in ((3, -1), (5, -1), (6, 0)):
        m = _map(occ, labels, 1, lift=lift)
        assert _at(m, 0, 0, "drop") == want, lift
    m = _map(occ, labels, 1, lift=6)
    assert _at(m, 0, 0, "support") == 4 and _at(m, 0, 0, "contacts") == 1
    assert _at(m, 1, 0, "drop") == 7 and _at(m, 1, 0, "support") == 3   # beside the shelf: down to the floor
    with pytest.raises(AssertionError):
        _map(occ, labels, 1, lift=7)                                    # the top leaves the grid


def _piece(mask):
    A, b = OB.grid_affine(T, DIM, EXT)
    return E.Piece(RO.pack(mask), DIM, RO.voxel_map(A, b), outside_keep=True)


def test_a_piece_lands_on_its_rest_only_when_the_rest_is_kept():
    occ, labels = _grid()
    _put(occ, labels, np.s_[0:2], 3)
    _put(occ, labels, np.s_[6:8, 4:6, 4:6], 1)                          # the piece
    _put(occ, labels, np.s_[2:4, 4:6, 4:6], 1)                          # the rest of label 1, below it
    mask = np.zeros((DIM,) * 3, dtype=bool)
    mask[6:8, 4:6, 4:6] = True
    piece = _piece(mask)
    keep = _map(occ, labels, 1, piece=piece)
    assert _at(keep, 0, 0, "drop") == 2 and _at(keep, 0, 0, "support") == 1
    drop = _map(occ, labels, 1, piece=piece, rest_drop=True)
    assert _at(drop, 0, 0, "drop") == 4 and _at(drop, 0, 0, "support") == 3
    assert keep["points"].shape[0] == drop["points"].shape[0] == 8


def test_without_anything_below_the_object_rests_unsupported_on_the_grid_floor():
    occ, labels = _grid()
    _put(occ, labels, np.s_[5:7, 4:7, 4:7], 1)
    _put(occ, labels, np.s_[9:11, 0:3, 0:3], 2)                         # above some offsets' columns: never below
    m = _map(occ, labels, 1)
    assert (m["support"] == -1).all() and (m["contacts"] == 0).all() and (m["drop"] == 5).all()
    m = _map(occ, labels, 1, lift=3)
    assert _at(m, -4, -4, "drop") == -1 and _at(m, 0, 0, "drop") == 8


def _scene(rng):
    """[h1, h2, y] with y up: a floor, random blocks of labels 2..5, and object 1 with overhangs."""
    g = np.zeros((DIM,) * 3, dtype=np.float32)
    lab = np.zeros((DIM,) * 3, dtype=np.int16)
    g[:, :, 0] = 0.9
    lab[:, :, 0] = 6
    for _ in range(12):
        a, b, c = rng.integers(0, DIM - 3, 3)
        g[a:a + 3, b:b + 2, c:c + 3] = 0.9
        lab[a:a + 3, b:b + 2, c:c + 3] = rng.integers(2, 6)
    g[5:8, 6:10, 12:14] = 0.9
    lab[5:8, 6:10, 12:14] = 1
    g[6, 6, 9:12] = 0.9
    lab[6, 6, 9:12] = 1
    return g, lab


def _posed(G, axis, sign):
    """The [h1, h2, y] grid G placed with its height along index axis `axis` (y = dim - 1 - idx when sign is +1)."""
    g = G[:, :, ::-1] if sign > 0 else G
    h = [a for a in range(3) if a != axis]
    order = [0, 0, 0]
    order[h[0]], order[h[1]], order[axis] = 0, 1, 2
    return np.ascontiguousarray(np.transpose(g, order))


def test_all_six_down_directions_give_the_same_map_on_a_permuted_grid():
    G, L = _scene(np.random.default_rng(5))
    A, _ = OB.grid_affine(T, DIM, EXT)
    maps = []
    for axis in range(3):
        for sign in (1, -1):
            occ, labels = _posed(G, axis, sign), _posed(L, axis, sign)
            down = sign * A[:, axis]
            assert PO.down_axis(T, EXT, down) == (axis, sign)
            for lift in (0, 2):
                maps.append((lift, _map(occ, labels, 1, lift=lift, down=down)))
    for lift in (0, 2):
        ref = next(m for l_, m in maps if l_ == lift)
        assert (ref["drop"] >= 0).any() and (ref["drop"] < 0).any() and (ref["support"] > 1).any()
        for l_, m in maps:
            if l_ == lift:
                for k in ("drop", "contacts", "support"):
                    np.testing.assert_array_equal(m[k], ref[k])
                assert m["offset_lo"] == ref["offset_lo"] and m["centre"] == ref["centre"]


def test_an_l_shape_overhanging_a_ledge_is_unstable_and_centred_is_stable():
    occ, labels = _grid()
    _put(occ, labels, np.s_[0:4, 0:8, :], 2)                            # the ledge: j 0..7, top at i 3
    _put(occ, labels, np.s_[10, 2:13, 6:9], 1)                          # a plate along j ...
    _put(occ, labels, np.s_[11:15, 12, 6:9], 1)                         # ... with an arm up at its far end
    m = _map(occ, labels, 1)
    assert m["centre"][0] == Fraction(33 * 7 + 12 * 12, 45)                 # (h1, h2) = (j, k)
    centred, over = (-2, 0), (2, 0)
    for (u, v), want in ((centred, True), (over, False)):
        cells = PO.support_cells(m, u, v)
        assert cells and {c[2] for c in cells} == {2} and max(c[0] for c in cells) == 7
        assert PO.stable(m, u, v) == want
        num = (m["centre"][0] * 45 + u * 45, m["centre"][1] * 45 + v * 45)
        assert OB.hull_contains([c[:2] for c in cells], num, 45) == want


def test_the_exact_hull_test_agrees_with_scipy():
    from scipy.spatial import ConvexHull
    rng = np.random.default_rng(11)
    checked = 0
    for _ in range(300):
        pts = rng.integers(-6, 7, (int(rng.integers(3, 12)), 2))
        try:
            hull = ConvexHull(pts)
        except Exception:                                                  # degenerate: covered by the exact cases below
            continue
        q = Fraction(int(rng.integers(-80, 81)), 10), Fraction(int(rng.integers(-80, 81)), 10)
        dist = (hull.equations[:, :2] @ np.array([float(q[0]), float(q[1])]) + hull.equations[:, 2]).max()
        if abs(dist) < 1e-9:
            continue
        want = bool(dist < 0)
        assert PO.in_hull(pts, q) == want
        assert OB.hull_contains(pts, (int(q[0] * 10), int(q[1] * 10)), 10) == want
        checked += 1
    assert checked > 200
    for cells, q, want in (([(0, 0)], (0, 0), True), ([(0, 0)], (Fraction(1, 3), 0), False),
                           ([(0, 0), (2, 2)], (1, 1), True), ([(0, 0), (2, 2)], (Fraction(5, 2), Fraction(5, 2)), False),
                           ([(0, 0), (2, 2)], (1, Fraction(3, 2)), False), ([(0, 0), (4, 0), (0, 4)], (2, 2), True),
                           ([(0, 0), (4, 0), (0, 4)], (Fraction(21, 10), 2), False), ([], (0, 0), False)):
        assert PO.in_hull(cells, q) == want
        den = q[0].denominator * q[1].denominator if isinstance(q[0], Fraction) and isinstance(q[1], Fraction) else 30
        assert OB.hull_contains(cells, (int(Fraction(q[0]) * den), int(Fraction(q[1]) * den)), den) == want


def test_the_transformation_follows_the_collision_checks_convention():
    """The placement's move equals slide_until_contact's on the same case, overlaps nothing, and one voxel lower overlaps."""
    step = EXT[0] / (DIM - 1)
    for gap in (0, 2, 5):
        occ, labels = _grid()
        _put(occ, labels, np.s_[0:2], 3)
        _put(occ, labels, np.s_[2 + gap:5 + gap, 4:7, 4:7], 1)
        m = _map(occ, labels, 1)
        d = int(m["drop"][4, 4])
        A, _ = OB.grid_affine(T, DIM, EXT)
        pm = {"horizontal": [1, 2], "axis": 0, "sign": -1, "lift": 0}
        delta = OB.placement_delta(pm, 0, 0, d)
        np.testing.assert_array_equal(delta, PO.delta(0, -1, 0, 0, 0, d))
        trans = OB.placement_transform(A, delta)
        dirn, s, mats = OB.slide_steps(UP_I, 8 * step, step)
        moves = [dict(label=1, trans=mt, box=(0, DIM - 1) * 3) for mt in mats]
        ov, _ = CO.move_overlap(occ, labels, T, EXT, moves, 0.45)
        r = OB.slide_result(dirn, s, [{"overlap": {}, "total": int(o.sum())} for o in ov], 0)
        np.testing.assert_allclose(trans, r["transformation"], rtol=0, atol=1e-15)
        lower = OB.placement_transform(A, OB.placement_delta(pm, 0, 0, d + 1))
        ov, _ = CO.move_overlap(occ, labels, T, EXT, [dict(label=1, trans=t, box=(0, DIM - 1) * 3) for t in (trans, lower)], 0.45)
        assert ov[0].sum() == 0 and ov[1].sum() > 0


def test_python_layer_rejects_bad_arguments():
    occ = torch.zeros((DIM,) * 3)
    lab = torch.zeros((DIM,) * 3, dtype=torch.int16)
    eye = np.eye(4)
    with pytest.raises(RuntimeError, match="CUDA"):
        OB.placement_map(occ, lab, eye, 1, (0, -1, 0))
    for kw, msg in ((dict(down=(0, 0, 0)), "down"), (dict(down=(np.nan, 1, 0)), "down"), (dict(down=(1, 0)), "down"),
                    (dict(lift=-1), "lift"), (dict(lift=1.5), "lift"), (dict(label=128), r"outside \[0, 127\]"),
                    (dict(label=-1), r"outside \[0, 127\]"), (dict(level=1.0), "level"), (dict(rest="x"), "rest"),
                    (dict(obstacles=[200]), "outside")):
        args = dict(label=1, down=(0, -1, 0))
        args.update(kw)
        with pytest.raises(ValueError, match=msg):
            OB.placement_map(occ, lab, eye, **args)
    for kw, msg in ((dict(near=(0, 0, np.inf)), "near"), (dict(near=(0, 0)), "near"), (dict(max_tests=0), "max_tests"),
                    (dict(on=[300]), "outside"), (dict(down=(0, 0, 0)), "down")):
        args = dict(label=1, down=(0, -1, 0), near=(0, 0, 0))
        args.update(kw)
        with pytest.raises(ValueError, match=msg):
            OB.place_object(occ, lab, eye, **args)


def test_move_objects_and_find_objects_check_the_placement_flags():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import find_objects
    import move_objects
    base = ["ck.tar", "--pose", "p.npy", "--hwk", "4", "4"] + ["1", "0", "2", "0", "1", "2", "0", "0", "1"] + \
        ["--move-label", "1", "--transform", "T.npy", "--out", "o"]
    a = move_objects.parse(base + ["--place-at", "0", "1", "2", "--down", "0", "-1", "0", "--on", "3", "4", "--lift", "2"])
    assert a.place_at == [0.0, 1.0, 2.0] and a.down == [0.0, -1.0, 0.0] and a.on == [3, 4] and a.lift == 2
    assert not a.any_stability and a.mode is None
    assert move_objects.parse(base + ["--place-at", "0", "0", "0", "--down", "0", "-1", "0", "--any-stability"]).any_stability
    place = ["--place-at", "0", "0", "0", "--down", "0", "-1", "0"]
    for extra, _msg in ((place + ["--until-contact"], "--until-contact"), (place + ["--distance", "0.1"], "--distance"),
                       (place + ["--yaw", "10"], "--yaw"), (place + ["--scale", "2"], "--scale"),
                       (place + ["--mode", "rotation"], "--mode"), (["--place-at", "0", "0", "0"], "--down"),
                       (place[:4] + ["--down", "0", "0", "0"], "down"), (place + ["--lift", "-1"], "lift"),
                       (["--mode", "translation", "--on", "2"], "--place-at"), (["--mode", "translation", "--lift", "1"], "--place-at"),
                       (["--mode", "translation", "--any-stability"], "--place-at"), ([], "--mode")):
        with pytest.raises(SystemExit):
            move_objects.parse(base + extra)
    a = find_objects.parse(["ck.tar", "--transform", "T.npy", "--placements", "3", "--down", "0", "-1", "0", "--out", "d"])
    assert a.placements == 3 and a.down == [0.0, -1.0, 0.0]
    with pytest.raises(SystemExit):
        find_objects.parse(["ck.tar", "--transform", "T.npy", "--placements", "3", "--down", "0", "-1", "0"])    # no --out
    for extra in (["--placements", "3"], ["--placements", "3", "--down", "0", "0", "0"], ["--placements", "128", "--down", "0", "1", "0"],
                  ["--placements", "3", "--down", "0", "1", "0", "--lift", "-2"], ["--lift", "2"]):
        with pytest.raises(SystemExit):
            find_objects.parse(["ck.tar", "--transform", "T.npy", "--out", "d"] + extra)
