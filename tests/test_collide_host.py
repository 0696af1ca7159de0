"""CPU: collision checks -- the numpy restatement of the rule (oracle/collide_oracle.py) on hand-built grids, the host stage of
slide_until_contact and supports, and the argument checks of the Python layer and of the tools (no GPU)."""
import os
import sys

import numpy as np
import pytest
import torch

from dmnerf_b200 import _lib
from dmnerf_b200 import objects as OB
from oracle import collide_oracle as CO
from oracle import edit_sweep_oracle as E
from oracle import region_oracle as RO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXT = (4.0, 4.0, 4.0)
DIM = 17                                             # grid points and 0.25 steps are exact in fp32
STEP = EXT[0] / (DIM - 1)


def _translate(x, y, z):
    m = np.eye(4)
    m[:3, 3] = (x, y, z)
    return m


def _move(label, trans, box=(0, DIM - 1) * 3, piece=None, rest_drop=False):
    return dict(label=label, trans=np.asarray(trans, dtype=np.float64), box=tuple(box), piece=piece, rest_drop=rest_drop)


def _cubes():
    """Label 1: a 3^3 cube at i 6..8; label 2: a 3^3 cube at i 10..12 (same j, k); label 3: a slab at i 0..1."""
    occ = np.zeros((DIM,) * 3, dtype=np.float32)
    labels = np.zeros((DIM,) * 3, dtype=np.int16)
    occ[6:9, 4:7, 4:7], labels[6:9, 4:7, 4:7] = 0.9, 1
    occ[10:13, 4:7, 4:7], labels[10:13, 4:7, 4:7] = 0.8, 2
    occ[0:2, :, :], labels[0:2, :, :] = 0.7, 3
    return occ, labels


def _check(occ, labels, moves, level=0.45, obstacles=None, T=np.eye(4)):
    ov, ld = CO.move_overlap(occ, labels, T, EXT, moves, level, obstacles)
    ov2, ld2 = CO.move_overlap(occ, labels, T, EXT, moves, level, obstacles, cull=False)
    np.testing.assert_array_equal(ov, ov2)
    np.testing.assert_array_equal(ld, ld2)
    return ov, ld


def test_identity_gives_no_overlap_and_the_full_landed():
    occ, labels = _cubes()
    for mv in (1, 2, 3):
        ov, ld = _check(occ, labels, [_move(mv, np.eye(4))])
        assert not ov.any() and ld[0] == np.count_nonzero((labels == mv) & (occ > 0.45))


def test_a_cube_moved_into_its_neighbour_overlaps_by_the_intersection():
    occ, labels = _cubes()
    for n in range(0, 7):
        # the object lands at inv(trans) x: translate by -n steps along the network x (= index i) moves it n voxels up in i
        ov, ld = _check(occ, labels, [_move(1, _translate(-n * STEP, 0, 0))])
        hi = min(8 + n, DIM - 1)
        inter = max(0, min(hi, 12) - max(6 + n, 10) + 1) * 9
        assert ld[0] == (hi - (6 + n) + 1) * 9                     # clipped at the grid face
        assert ov[0, 2] == inter and ov[0].sum() == inter, n


def test_a_scale_of_two_lands_eight_times_the_voxels():
    occ = np.zeros((DIM,) * 3, dtype=np.float32)
    labels = np.zeros((DIM,) * 3, dtype=np.int16)
    occ[8:10, 8:10, 8:10], labels[8:10, 8:10, 8:10] = 0.9, 5
    c = E.sweep_points(np.eye(4), EXT, DIM).reshape(DIM, DIM, DIM, 3)[8, 8, 8].astype(np.float64)
    trans = _translate(*c) @ np.diag([0.5, 0.5, 0.5, 1.0]) @ _translate(*-c)    # lands at 2 (x - c) + c
    ov, ld = _check(occ, labels, [_move(5, trans)])
    # p lands when rint(c + (p - c) / 2) in 8..9: p - c in -1 .. 3 (half to even), 4 points per axis
    q = np.rint(8 + (np.arange(DIM) - 8) / 2.0)
    per_axis = int(np.count_nonzero((q >= 8) & (q <= 9)))
    assert ld[0] == per_axis ** 3 and not ov.any()


def _piece(mask):
    A, b = OB.grid_affine(np.eye(4), DIM, EXT)
    return E.Piece(RO.pack(mask), DIM, RO.voxel_map(A, b), outside_keep=True)


def test_a_piece_collides_with_its_own_rest_only_when_the_rest_is_kept():
    occ = np.zeros((DIM,) * 3, dtype=np.float32)
    labels = np.zeros((DIM,) * 3, dtype=np.int16)
    occ[4:6, 4:6, 4:6], labels[4:6, 4:6, 4:6] = 0.9, 1                 # the piece
    occ[8:10, 4:6, 4:6], labels[8:10, 4:6, 4:6] = 0.9, 1               # the rest of label 1, 4 voxels up in i
    mask = np.zeros((DIM,) * 3, dtype=bool)
    mask[4:6, 4:6, 4:6] = True
    piece = _piece(mask)
    trans = _translate(-4 * STEP, 0, 0)
    ov, ld = _check(occ, labels, [_move(1, trans, piece=piece), _move(1, trans, piece=piece, rest_drop=True)])
    assert ld.tolist() == [8, 8]
    assert ov[0, 1] == 8 and ov[0].sum() == 8
    assert not ov[1].any()
    # the piece does not collide with the points it vacates
    ov, _ = _check(occ, labels, [_move(1, _translate(-1 * STEP, 0, 0), piece=piece)])
    assert not ov.any()


def test_the_obstacle_mask_leaves_labels_out():
    occ, labels = _cubes()
    trans = _translate(-3 * STEP, 0, 0)
    ov, _ = _check(occ, labels, [_move(1, trans)])
    assert ov[0, 2] > 0
    ov, _ = _check(occ, labels, [_move(1, trans)], obstacles=[3])
    assert not ov.any()


def test_culling_never_changes_a_count():
    rng = np.random.default_rng(7)
    occ = (rng.random((DIM,) * 3) > 0.6).astype(np.float32)
    labels = rng.integers(0, 4, (DIM,) * 3).astype(np.int16)
    moves = []
    for k in range(12):
        a = rng.normal(size=3)
        a /= np.linalg.norm(a)
        ang = rng.uniform(-np.pi, np.pi)
        K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
        m = np.eye(4)
        m[:3, :3] = (np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K) * rng.uniform(0.6, 1.6)
        m[:3, 3] = rng.uniform(-1.5, 1.5, 3)
        lo = rng.integers(0, DIM // 2, 3)
        box = [v for a_ in range(3) for v in (int(lo[a_]), int(lo[a_] + rng.integers(1, DIM // 2)))]
        moves.append(_move(int(rng.integers(0, 4)), m, box))
    T = np.eye(4)
    T[:3, :3] = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    T[:3, 3] = (0.3, -0.1, 0.2)
    for t in (np.eye(4), T):
        ov, ld = _check(occ, labels, moves, T=t)
        assert ld.sum() > 0 and ov.sum() > 0


def test_an_object_above_a_slab_slides_exactly_the_gap():
    occ, labels = _cubes()
    for gap in (0, 1, 3):
        occ2, lab2 = occ.copy(), labels.copy()
        occ2[labels == 1] = 0.0
        occ2[2 + gap:5 + gap, 4:7, 4:7], lab2[2 + gap:5 + gap, 4:7, 4:7] = 0.9, 1    # `gap` empty voxels above the slab
        d, s, mats = OB.slide_steps((-1.0, 0.0, 0.0), 6 * STEP, STEP)
        ov, ld = _check(occ2, lab2, [_move(1, m) for m in mats])
        results = [{"overlap": {int(k): int(ov[i, k]) for k in np.nonzero(ov[i])[0]}, "total": int(ov[i].sum())}
                   for i in range(len(mats))]
        r = OB.slide_result(d, s, results, 0)
        assert r["distance"] == pytest.approx(gap * STEP) and r["contact"]["distance"] == pytest.approx((gap + 1) * STEP)
        assert r["contact"]["overlap"] == {3: 9} and r["profile"][gap + 1] == 9
        assert np.allclose(r["transformation"], _translate(gap * STEP, 0, 0))
        r = OB.slide_result(d, s, results, 9)                      # tolerating one layer
        assert r["distance"] == pytest.approx(min(gap + 1, 6) * STEP)
    r = OB.slide_result(d, s, [{"overlap": {}, "total": 0}] * len(s), 0)
    assert r["distance"] == 6 * STEP and r["contact"] is None
    r = OB.slide_result(d, s, [{"overlap": {3: 1}, "total": 1}] * len(s), 0)
    assert r["distance"] is None and r["transformation"] is None and r["contact"]["distance"] == 0.0


def test_slide_steps_end_at_max_distance_and_are_capped():
    d, s, mats = OB.slide_steps((0.0, 3.0, 0.0), 1.0, 0.3)
    assert d.tolist() == [0.0, 1.0, 0.0] and s.tolist() == pytest.approx([0.0, 0.3, 0.6, 0.9, 1.0])
    assert np.allclose(mats[2], _translate(0.0, -0.6, 0.0))
    base = _translate(1.0, 0.0, 0.0)
    _, _, mats = OB.slide_steps((0.0, 1.0, 0.0), 1.0, 0.5, base)
    assert np.allclose(mats[1], base @ _translate(0.0, -0.5, 0.0))
    assert len(OB.slide_steps((1, 0, 0), _lib.MAX_CANDIDATES - 1, 1.0)[1]) == _lib.MAX_CANDIDATES
    with pytest.raises(ValueError, match="exceed"):
        OB.slide_steps((1, 0, 0), _lib.MAX_CANDIDATES, 1.0)


def test_face_contacts_and_supports_under_a_quarter_turn():
    occ = np.zeros((8, 8, 8), dtype=np.float32)
    labels = np.zeros((8, 8, 8), dtype=np.int16)
    occ[2:4, 2:5, 2:6], labels[2:4, 2:5, 2:6] = 0.9, 4                 # sits on top of ...
    occ[4:6, 2:5, 2:6], labels[4:6, 2:5, 2:6] = 0.9, 7                 # ... this one, along +i
    occ[7, :, :], labels[7, :, :] = 0.9, 9                              # not touching: row 6 is empty
    faces = CO.object_contacts(occ, labels, 0.45)
    assert faces[0, 4, 7] == 12 and faces[0, 7, 4] == 0 and faces.sum() == 12
    # a quarter turn of the grid about the mesh z axis: index i runs along the mesh +y, which is the network +z
    T = np.eye(4)
    T[:3, :3] = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    c = OB.contacts_from_faces(faces, T, 8, EXT)
    np.testing.assert_allclose(c["axes"], [[0, 0, 1], [-1, 0, 0], [0, -1, 0]], atol=1e-15)
    np.testing.assert_allclose(c["face_area"], [(4 / 7) ** 2] * 3)
    down = np.array([0.0, 0.0, 1.0])                                     # +i points down: 4 is above 7
    assert OB.supports(c, down) == {4: [(7, 12)]}
    assert OB.supports(c, -down) == {7: [(4, 12)]}
    assert OB.supports(c, down + 0.3 * c["axes"][1]) == {4: [(7, 12)]}
    assert OB.supports(c, down, min_faces=13) == {}
    assert OB.supports(c, c["axes"][1]) == {}


def test_python_layer_rejects_bad_arguments():
    occ = torch.zeros((DIM,) * 3)
    lab = torch.zeros((DIM,) * 3, dtype=torch.int16)
    eye = np.eye(4)
    with pytest.raises(RuntimeError, match="CUDA"):
        OB.move_overlap(occ, lab, eye, [(1, eye)])
    with pytest.raises(RuntimeError, match="CUDA"):
        OB.object_contacts(occ, lab, eye)
    with pytest.raises(ValueError, match="tolerance"):
        OB.slide_until_contact(occ, lab, eye, 1, (1, 0, 0), 1.0, tolerance=-1)
    with pytest.raises(ValueError, match="tolerance"):
        OB.slide_until_contact(occ, lab, eye, 1, (1, 0, 0), 1.0, tolerance=0.5)
    with pytest.raises(ValueError, match="direction"):
        OB.slide_until_contact(occ, lab, eye, 1, (0, 0, 0), 1.0)
    bad = [
        (dict(direction=(0, 0, 0)), "direction"),
        (dict(direction=(np.nan, 0, 0)), "direction"),
        (dict(max_distance=-1.0), "max_distance"),
        (dict(step=0.0), "step"),
        (dict(max_distance=1e9, step=1.0), "exceed"),
        (dict(base=np.diag([1.0, -1.0, 1.0, 1.0])), "determinant"),
    ]
    for kw, msg in bad:
        args = dict(direction=(1, 0, 0), max_distance=1.0, step=0.1)
        args.update(kw)
        with pytest.raises(ValueError, match=msg):
            OB.slide_steps(**args)
    with pytest.raises(ValueError, match="down"):
        OB.supports({"axes": np.eye(3), "faces": np.zeros((3, 128, 128))}, (0, 0, 0))
    with pytest.raises(ValueError, match="min_faces"):
        OB.supports({"axes": np.eye(3), "faces": np.zeros((3, 128, 128))}, (1, 0, 0), min_faces=0)
    with pytest.raises(ValueError, match="at most 4096"):
        OB._check_moves([(1, eye)] * 4097, 127, _lib.MAX_CANDIDATES)
    assert len(OB._check_moves([(1, eye)] * 4096, 127, _lib.MAX_CANDIDATES)[0]) == 4096
    with pytest.raises(ValueError, match="at most 8"):
        OB._check_moves([(1, eye)] * 9, 127)


def test_move_objects_and_find_objects_check_their_flags():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import find_objects
    import move_objects
    base = ["ck.tar", "--pose", "p.npy", "--hwk", "4", "4"] + ["1", "0", "2", "0", "1", "2", "0", "0", "1"] + [ "--move-label", "1", "--transform", "T.npy", "--out", "o"]
    a = move_objects.parse(base + ["--mode", "translation", "--until-contact", "--check"])
    assert a.until_contact and a.check and a.step is None and a.tolerance == 0
    a = move_objects.parse(base + ["--mode", "rotation"])
    assert not a.until_contact and not a.check
    for extra, msg in ((["--mode", "rotation", "--until-contact"], "translation"),
                       (["--mode", "translation", "--until-contact", "--distance", "0"], "distance"),
                       (["--mode", "translation", "--step", "0.1"], "--until-contact"),
                       (["--mode", "translation", "--until-contact", "--step", "0"], "step"),
                       (["--mode", "translation", "--until-contact", "--tolerance", "-1"], "tolerance")):
        with pytest.raises(SystemExit):
            move_objects.parse(base + extra)
    a = find_objects.parse(["ck.tar", "--transform", "T.npy", "--contacts", "--down", "0", "-1", "0"])
    assert a.contacts and a.down == [0.0, -1.0, 0.0]
    with pytest.raises(SystemExit):
        find_objects.parse(["ck.tar", "--transform", "T.npy", "--down", "0", "-1", "0"])
    with pytest.raises(SystemExit):
        find_objects.parse(["ck.tar", "--transform", "T.npy", "--contacts", "--down", "0", "0", "0"])
