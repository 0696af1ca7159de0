"""GPU: collision checks -- dmnerf_move_overlap and dmnerf_object_contacts against the numpy rule (oracle/collide_oracle.py) on
synthetic keep-all sweeps, the agreement with edited_sweep on an exact grid, slide_until_contact, the rejections and the tools'
--check / --until-contact / --contacts."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from dmnerf_b200 import _lib
from dmnerf_b200 import objects as OB
from dmnerf_b200.engine import get_context
from dmnerf_b200.testing import make_models
from oracle import collide_oracle as CO
from oracle import edit_sweep_oracle as E

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
QUANTILE = 0.5                       # the synthetic networks need not cross 0.45: each test's level is a quantile of its sweep
NEAR, FAR, NI = 4.0, 15.0, 128
EXACT = dict(T=np.eye(4), dim=33, ext=(4.0, 4.0, 4.0))      # grid points and 0.125 steps are exact in fp32


@pytest.fixture(scope="module", params=[13, 93])
def nets(request):
    return make_models(101, 202, request.param, DEV)


def _sweep(nf, T, dim, ext):
    ins_num = int(nf.ins_linear.weight.shape[0]) - 1
    return OB.occupancy_objects(nf, T, OB.object_mask(ins_num, remove=[]), dim, ext, NEAR, FAR, NI, device=DEV)


def _level(occ):
    x = occ.flatten().float()
    x = x[x > 0]
    lv = float(x.kthvalue(max(1, int(QUANTILE * x.numel()))).values)
    assert 0.0 < lv < 1.0
    return lv


def _np(*ts):
    return [t.cpu().numpy() for t in ts]


def _solid_labels(occ, labels, lv, n=3):
    lab = labels[occ > np.float32(lv)]
    k, c = np.unique(lab, return_counts=True)
    return [int(x) for x in k[np.argsort(-c, kind="stable")][:n]]


def _translate(v):
    m = np.eye(4)
    m[:3, 3] = v
    return m


def _turn_about(c, k=1):
    R = np.linalg.matrix_power(np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]]), k)
    m = np.eye(4)
    m[:3, :3] = R
    m[:3, 3] = np.asarray(c) - R @ np.asarray(c)
    return m


def _oracle(o, l, T, ext, moves, boxes, lv, pieces=None, rest="keep", obstacles=None, cull=False):
    drops = [rest == "drop"] * len(moves)
    pc = [None if p is None else E.Piece(p.bits.cpu().numpy(), p.dim, p.voxel_map, p.outside == "keep")
          for p in (pieces or [None] * len(moves))]
    mv = [dict(label=k, trans=np.asarray(m, dtype=np.float64), box=tuple(int(v) for v in b), piece=p, rest_drop=d)
          for (k, m), b, p, d in zip(moves, boxes, pc, drops)]
    return CO.move_overlap(o, l, T, ext, mv, lv, obstacles, cull)


def _assert_equal(got, want):
    ov, ld = want
    assert [r["landed"] for r in got] == ld.tolist()
    for r, row in zip(got, ov):
        assert r["overlap"] == {int(k): int(row[k]) for k in np.nonzero(row)[0]} and r["total"] == int(row.sum())


# ---- 1. against the numpy rule ------------------------------------------------------------------------------------------------

def test_exact_grid_moves_pieces_and_obstacles_equal_the_rule(nets):
    _, nf, _, _ = nets
    T, dim, ext = EXACT["T"], EXACT["dim"], EXACT["ext"]
    occ, lab = _sweep(nf, T, dim, ext)
    lv = _level(occ)
    o, l = _np(occ, lab)
    top = _solid_labels(o, l, lv)
    c = np.array([0.125 * 3, -0.125 * 2, 0.0])
    moves = [(top[0], np.eye(4)), (top[0], _translate((0.125 * 3, 0.0, -0.125 * 2))), (top[1 % len(top)], _turn_about(c, 1)),
             (top[2 % len(top)], _translate((-0.25, 0.125, 0.375)) @ _turn_about(c, 2))]
    boxes = OB.edit_boxes(occ, lab, moves, T, ext, lv)
    got = OB.move_overlap(occ, lab, T, moves, ext, lv)
    _assert_equal(got, _oracle(o, l, T, ext, moves, boxes, lv))
    assert got[0]["total"] == 0 and got[0]["landed"] == int(((l == top[0]) & (o > lv)).sum())    # the identity
    obst = [k for k in range(OB.MAX_LABELS) if k % 2]
    _assert_equal(OB.move_overlap(occ, lab, T, moves, ext, lv, obstacles=obst), _oracle(o, l, T, ext, moves, boxes, lv, obstacles=obst))
    cc = OB.object_components(occ, lab, lv, 26)
    piece = OB.component_region(cc, [OB.largest_components(cc["label"], cc["voxels"])[top[0]]], T, ext)
    pm = [(top[0], np.eye(4)), (top[0], _translate((0.25, 0.0, -0.125)))]
    for rest in ("keep", "drop"):
        got = OB.move_overlap(occ, lab, T, pm, ext, lv, pieces=[piece] * 2, rest=rest)
        want = _oracle(o, l, T, ext, pm, OB.edit_boxes(occ, lab, pm, T, ext, lv, 2, [piece] * 2), lv, [piece] * 2, rest)
        _assert_equal(got, want)
        assert got[0]["total"] == 0


@pytest.mark.parametrize("mode", ["rotation", "scale", "multi"])
def test_off_grid_moves_equal_the_rule(nets, golden_dir, mode):
    _, nf, _, _ = nets
    g = np.load(os.path.join(golden_dir, "mesh_grid.npz"))
    T, dim, ext = g["transform_a"], 40, g["extents"]
    occ, lab = _sweep(nf, T, dim, ext)
    lv = _level(occ)
    o, l = _np(occ, lab)
    A, b = OB.grid_affine(T, dim, ext)
    trans = OB.manipulation_transform(A @ np.full(3, (dim - 1) / 2.0) + b, mode)["transformations"][0]["transformation"]
    moves = [(k, trans) for k in _solid_labels(o, l, lv)]
    boxes = OB.edit_boxes(occ, lab, moves, T, ext, lv)
    got = OB.move_overlap(occ, lab, T, moves, ext, lv)
    _assert_equal(got, _oracle(o, l, T, ext, moves, boxes, lv))
    assert sum(r["landed"] for r in got) > 0


def test_one_and_4096_candidates_and_culling_against_the_whole_grid(nets):
    _, nf, _, _ = nets
    T, dim, ext = EXACT["T"], EXACT["dim"], EXACT["ext"]
    occ, lab = _sweep(nf, T, dim, ext)
    lv = _level(occ)
    lab[dim // 2:] = (lab[dim // 2:] + 1) % OB.MAX_LABELS      # a second object, so that the moves meet other labels
    o, l = _np(occ, lab)
    top = _solid_labels(o, l, lv)
    rng = np.random.default_rng(3)
    moves = []
    for i in range(_lib.MAX_CANDIDATES):
        a = rng.normal(size=3)
        q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        q *= np.sign(np.linalg.det(q))
        m = np.eye(4)
        m[:3, :3] = q * rng.uniform(0.7, 1.4) if i % 2 else np.eye(3)
        m[:3, 3] = 0.125 * np.rint(4 * a) if i % 2 == 0 else a * 0.5
        moves.append((top[i % len(top)], m))
    boxes = OB.edit_boxes(occ, lab, moves[:len(top)], T, ext, lv)
    boxes = np.asarray([boxes[i % len(top)] for i in range(len(moves))])
    got = OB.move_overlap(occ, lab, T, moves, ext, lv, boxes=boxes)
    assert got == OB.move_overlap(occ, lab, T, moves, ext, lv, boxes=boxes)               # bit-reproducible
    assert sum(r["total"] > 0 for r in got) > 100
    _assert_equal(got, _oracle(o, l, T, ext, moves, boxes, lv, cull=True))
    sub = list(range(0, len(moves), 97))
    _assert_equal([got[i] for i in sub], _oracle(o, l, T, ext, [moves[i] for i in sub], boxes[sub], lv, cull=False))
    one = OB.move_overlap(occ, lab, T, moves[1:2], ext, lv, boxes=boxes[1:2])
    assert one == got[1:2]


# ---- 2. agreement with the edit ------------------------------------------------------------------------------------------------

def test_overlap_is_what_edited_sweep_overwrites_on_the_exact_grid(nets):
    _, nf, _, _ = nets
    T, dim, ext = EXACT["T"], EXACT["dim"], EXACT["ext"]
    occ, lab = _sweep(nf, T, dim, ext)
    lv = _level(occ)
    o, l = _np(occ, lab)
    for mv, trans in [(k, _translate(v)) for k, v in zip(_solid_labels(o, l, lv), [(0.375, 0, -0.25), (0, -0.5, 0.125),
                                                                                   (-0.25, 0.25, 0.0)])]:
        r = OB.move_overlap(occ, lab, T, [(mv, trans)], ext, lv)[0]
        eo, el = _np(*OB.edited_sweep(nf, T, [(mv, trans)], dim, ext, lv, NEAR, FAR, NI))
        landed_solid = (el == mv) & (eo > lv)
        over = (o > lv) & (l != mv) & landed_solid
        want = {int(k): int(c) for k, c in zip(*np.unique(l[over], return_counts=True))}
        assert r["overlap"] == want and r["total"] == int(over.sum())
        assert r["landed"] == int(landed_solid.sum())


# ---- 3. sliding --------------------------------------------------------------------------------------------------------------

def test_slide_until_contact_stops_before_the_first_overlap(nets):
    _, nf, _, _ = nets
    T, dim, ext = EXACT["T"], EXACT["dim"], EXACT["ext"]
    occ, lab = _sweep(nf, T, dim, ext)
    lv = _level(occ)
    o, l = _np(occ, lab)
    contacts = 0
    for mv in _solid_labels(o, l, lv):
        for direction, tol, base in (((0.0, -1.0, 0.0), 0, None), ((1.0, 0.0, 0.0), 0, None),
                                     ((0.0, 0.0, 1.0), 5, _translate((0.0, 0.0, 0.125)))):
            r = OB.slide_until_contact(occ, lab, T, mv, direction, 4.0, base=base, tolerance=tol, extents=ext, level=lv)
            assert r["steps"][1] == 0.125 and len(r["steps"]) == len(r["profile"]) == 33
            if r["distance"] is None:
                assert r["profile"][0] > tol and r["contact"]["distance"] == 0.0
                continue
            k = r["steps"].index(r["distance"])
            assert max(r["profile"][:k + 1]) <= tol
            if r["contact"] is not None:
                contacts += 1
                assert r["profile"][k + 1] > tol and r["contact"]["distance"] == r["steps"][k + 1]
            eo, el = _np(*OB.edited_sweep(nf, T, [(mv, r["transformation"])], dim, ext, lv, NEAR, FAR, NI))
            overwritten = (o > lv) & (l != mv) & (el == mv) & (eo > lv)
            assert int(overwritten.sum()) == r["profile"][k] <= tol
    assert contacts > 0 or len(_solid_labels(o, l, lv)) == 1                  # one solid label: nothing to meet


# ---- 4. contacts ---------------------------------------------------------------------------------------------------------------

def test_object_contacts_equal_numpy(nets, golden_dir):
    _, nf, _, _ = nets
    g = np.load(os.path.join(golden_dir, "mesh_grid.npz"))
    T, dim, ext = g["transform_a"], 48, g["extents"]
    occ, lab = _sweep(nf, T, dim, ext)
    lv = _level(occ)
    c = OB.object_contacts(occ, lab, T, ext, lv)
    np.testing.assert_array_equal(c["faces"], CO.object_contacts(*_np(occ, lab), lv))
    np.testing.assert_array_equal(OB.object_contacts(occ, lab, T, ext, lv)["faces"], c["faces"])
    rng = np.random.default_rng(1)
    ro = torch.from_numpy(rng.random((37, 37, 37)).astype(np.float32)).to(DEV)
    rl = torch.from_numpy(rng.integers(0, 128, (37, 37, 37)).astype(np.int16)).to(DEV)
    faces = OB.object_contacts(ro, rl, T, ext, 0.45)["faces"]
    np.testing.assert_array_equal(faces, CO.object_contacts(*_np(ro, rl), 0.45))
    assert faces.sum() > 0


# ---- 5. rejections -----------------------------------------------------------------------------------------------------------

def test_the_library_rejects_bad_input():
    dim, lv = 8, 0.45
    occ = torch.zeros((dim,) * 3, device=DEV)
    lab = torch.zeros((dim,) * 3, device=DEV, dtype=torch.int16)
    ctx = get_context(DEV)

    def overlap(n=1, label=1, trans=np.eye(4), box=(0, dim - 1) * 3, level=lv, d=dim, o=occ, la=lab):
        arr = (_lib.EditMove * max(1, n))()
        for i in range(n):
            arr[i].label = label
            arr[i].trans[:] = list(np.asarray(trans, dtype=np.float64)[:3].reshape(-1))
            arr[i].box[:] = list(box)
        ov = np.zeros((max(1, n), 128), dtype=np.int64)
        ld = np.zeros(max(1, n), dtype=np.int64)
        with pytest.raises(RuntimeError) as e:
            ctx.call("dmnerf_move_overlap", ctx.handle, _lib.ptr(o), _lib.ptr(la, torch.int16), d, level, _lib.doubles(np.eye(4), 16),
                     _lib.doubles((4.0, 4.0, 4.0), 3), arr, n, None, ov.ctypes.data_as(C.POINTER(C.c_int64)),
                     ld.ctypes.data_as(C.POINTER(C.c_int64)))
        assert not ov.any() and not ld.any()
        return str(e.value)

    def contacts(n_labels=128, level=lv, d=dim, o=occ, la=lab):
        f = np.zeros((3, max(1, n_labels), max(1, n_labels)), dtype=np.int64)
        with pytest.raises(RuntimeError) as e:
            ctx.call("dmnerf_object_contacts", ctx.handle, _lib.ptr(o), _lib.ptr(la, torch.int16), d, level, n_labels,
                     f.ctypes.data_as(C.POINTER(C.c_int64)))
        assert not f.any()
        return str(e.value)

    assert "between 1 and 4096" in overlap(n=0)
    assert "between 1 and 4096" in overlap(n=4097)
    assert "outside [0, 127]" in overlap(label=128)
    assert "det" in overlap(trans=np.diag([1.0, -1.0, 1.0, 1.0]))
    assert "not finite" in overlap(trans=np.full((4, 4), np.nan))
    assert "inverted or outside" in overlap(box=(0, dim, 0, 1, 0, 1))
    assert "level" in overlap(level=0.0) and "level" in overlap(level=1.0)
    assert "dim" in overlap(d=1) and "dim" in overlap(d=2049)
    bad = lab.clone()
    bad[3, 4, 5] = 128
    assert "label outside [0, 127]" in overlap(la=bad)
    nan = occ.clone()
    nan[1, 2, 3] = float("nan")
    assert "NaN" in overlap(o=nan)
    assert "n_labels" in contacts(n_labels=0) and "n_labels" in contacts(n_labels=129)
    assert "dim" in contacts(d=1) and "level" in contacts(level=1.0)
    small = lab.clone()
    small[0, 0, 0] = 5
    assert "label outside [0, 4]" in contacts(n_labels=5, la=small)
    assert "label outside [0, 3]" in contacts(n_labels=4, la=small)
    assert "NaN" in contacts(o=nan)
    with pytest.raises(ValueError, match="outside"):
        OB.move_overlap(occ, lab, np.eye(4), [(128, np.eye(4))], (4.0, 4.0, 4.0))
    with pytest.raises(ValueError, match="level"):
        OB.move_overlap(occ, lab, np.eye(4), [(1, np.eye(4))], (4.0, 4.0, 4.0), level=1.5)
    with pytest.raises(ValueError, match="int16"):
        OB.object_contacts(occ, lab.int(), np.eye(4), (4.0, 4.0, 4.0))
    with pytest.raises(ValueError, match="exceed"):
        OB.slide_until_contact(occ, lab, np.eye(4), 1, (1, 0, 0), 1e6, extents=(4.0, 4.0, 4.0))


# ---- 6. tools ----------------------------------------------------------------------------------------------------------------

def _checkpoint(tmp_path):
    nc, nf, _, _ = make_models(7, 8, 13, "cpu", trained_like=True)
    torch.save({"network_coarse_state_dict": nc.state_dict(), "network_fine_state_dict": nf.state_dict()}, tmp_path / "ck.tar")
    np.save(tmp_path / "T.npy", np.eye(4))
    return make_models(7, 8, 13, DEV, trained_like=True)[1]


def test_move_objects_check_and_until_contact_write_what_the_library_returns(tmp_path):
    nf = _checkpoint(tmp_path)
    pose = np.eye(4, dtype=np.float32)
    pose[2, 3] = 6.0
    np.save(tmp_path / "pose.npy", pose)
    ext = (1.9, 7.0, 7.0)
    o, l = _np(*OB.occupancy_objects(nf, np.eye(4), OB.object_mask(13, keep=range(13)), 32, ext, device=DEV))
    lv = _level(torch.from_numpy(o))
    label = _solid_labels(o, l, lv, 1)[0]
    argv = [str(tmp_path / "ck.tar"), "--pose", str(tmp_path / "pose.npy"), "--hwk", "24", "32", "30", "0", "16", "0", "30", "12", "0",
            "0", "1", "--move-label", str(label), "--mode", "translation", "--distance", "0.8", "--transform", str(tmp_path / "T.npy"),
            "--grid-dim", "32", "--level", repr(lv), "--out", str(tmp_path / "o"), "--N-test", "256", "--check", "--until-contact"]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "move_objects.py")] + argv, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    info = json.loads(r.stdout.strip().splitlines()[-1])
    with open(tmp_path / "o" / "transform.json") as fh:
        assert json.load(fh) == {k: v for k, v in info.items() if k != "files"}
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import move_objects
    a = move_objects.parse(argv)
    _, lab_, centre, region = move_objects.choose_piece(a, nf, np.eye(4), ext)
    occ, lab = OB.occupancy_objects(nf, np.eye(4), OB.object_mask(13, remove=[]), 32, ext, device=DEV)
    s = OB.slide_until_contact(occ, lab, np.eye(4), lab_, (0.0, -1.0, 0.0), 0.8, extents=ext, level=lv, piece=region)
    assert info["slide"]["requested"] == 0.8 and info["slide"]["found"] == s["distance"]
    assert (info["slide"]["contact"] is None) == (s["contact"] is None)
    trans = OB.manipulation_transform(centre, "translation", distance=s["distance"] or 0.0)["transformations"]
    np.testing.assert_allclose(info["transformations"][0]["transformation"], trans[0]["transformation"], rtol=0, atol=0)
    c = OB.move_overlap(occ, lab, np.eye(4), [(lab_, trans[0]["transformation"])], ext, lv, pieces=[region])[0]
    assert info["landed"] == c["landed"] and info["overlap"]["voxels"] == {str(k): v for k, v in c["overlap"].items()}


def test_find_objects_contacts_write_what_the_library_returns(tmp_path):
    nf = _checkpoint(tmp_path)
    ext = (1.9, 7.0, 7.0)
    occ, lab = OB.occupancy_objects(nf, np.eye(4), OB.object_mask(13, keep=range(13)), 32, ext, device=DEV)
    lv = _level(occ)
    base = [sys.executable, os.path.join(ROOT, "tools", "find_objects.py"), str(tmp_path / "ck.tar"), "--transform",
            str(tmp_path / "T.npy"), "--grid-dim", "32", "--level", repr(lv)]
    r = subprocess.run(base + ["--contacts", "--down", "0", "-1", "0"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    info = json.loads(r.stdout.strip().splitlines()[-1])
    plain = subprocess.run(base, capture_output=True, text=True)
    assert plain.returncode == 0, plain.stderr[-3000:]
    plain = json.loads(plain.stdout.strip().splitlines()[-1])
    assert [{k: v for k, v in e.items() if k != "rests_on"} for e in info["objects"]] == plain["objects"]
    c = OB.object_contacts(occ, lab, np.eye(4), ext, lv)
    pairs = {(p["axis"], p["labels"][0], p["labels"][1]): p["faces"] for p in info["contacts"]["pairs"]}
    assert pairs == {(int(a), int(x), int(y)): int(c["faces"][a, x, y]) for a, x, y in zip(*np.nonzero(c["faces"]))}
    below = OB.supports(c, (0, -1, 0))
    for e in info["objects"]:
        assert e["rests_on"] == [{"label": k, "faces": n} for k, n in below.get(e["label"], [])]
