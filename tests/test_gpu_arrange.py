"""GPU: arranging objects -- dmnerf_grid_edit, the _in_scene placement maps and arrange_objects against the numpy rule
(oracle/arrange_oracle.py) on synthetic keep-all sweeps and hand-built grids, the single-move counts against dmnerf_move_overlap,
the exact-grid agreement with edited_sweep, repeatability, the rejections and tools/move_objects.py --arrange."""
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
from oracle import arrange_oracle as AO
from oracle import edit_sweep_oracle as E
from oracle import placement_oracle as PO
from oracle import placement_turn_oracle as TO

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
NEAR, FAR, NI = 4.0, 15.0, 128
T, DIM, EXT = np.eye(4), 33, (4.0, 4.0, 4.0)       # grid points and 0.125 steps are exact in fp32
DOWN = (0.0, -1.0, 0.0)


@pytest.fixture(scope="module", params=[13, 93])
def nets(request):
    return make_models(101, 202, request.param, DEV)


def _sweep(nf, dim=DIM):
    ins_num = int(nf.ins_linear.weight.shape[0]) - 1
    return OB.occupancy_objects(nf, T, OB.object_mask(ins_num, remove=[]), dim, EXT, NEAR, FAR, NI, device=DEV)


def _level(occ, q=0.5):
    """A quantile of the sweep's occupancy: the synthetic networks need not cross 0.45."""
    x = occ.flatten().float()
    x = x[x > 0]
    return float(x.kthvalue(max(1, int(q * x.numel()))).values)


def _np(*ts):
    return [t.cpu().numpy() for t in ts]


def _labels_by_size(o, l, lv, n):
    """n labels with solid points, most points first (repeated when the sweep has fewer)."""
    k, c = np.unique(l[o > np.float32(lv)], return_counts=True)
    k = [int(x) for x in k[np.argsort(-c, kind="stable")][:n]]
    return [k[i % len(k)] for i in range(n)]


def _centre(o, l, lv, label):
    idx = np.argwhere((l == label) & (o > np.float32(lv)))
    return idx.mean(0)


def _turn(angle, about):
    """A turn by `angle` degrees about the network x axis through the network point `about`, as a move."""
    c, s = OB._turn_cos_sin(angle)
    R = np.eye(4)
    R[1:3, 1:3] = [[c, -s], [s, c]]
    P = np.eye(4)
    P[:3, 3] = about
    Q = np.eye(4)
    Q[:3, 3] = -np.asarray(about)
    return P @ R @ Q


def _oracle_moves(o, l, lv, moves, pieces=None, rest="keep", boxes=None):
    out = []
    for i, (k, m) in enumerate(moves):
        p = None if pieces is None or pieces[i] is None else E.Piece(pieces[i].bits.cpu().numpy(), pieces[i].dim, pieces[i].voxel_map,
                                                                    pieces[i].outside == "keep")
        keep = None if p is None else p.keeps(E.sweep_points(T, EXT, o.shape[0])).reshape(o.shape)
        box = E.solid_box(o, l, k, lv, 2, keep) if boxes is None else boxes[i]
        out.append({"label": k, "trans": np.asarray(m, dtype=np.float64), "box": box, "piece": p,
                    "rest_drop": (rest if isinstance(rest, str) else rest[i]) == "drop"})
    return out


def _check_edit(occ, lab, lv, moves, pieces=None, rest="keep", boxes=None):
    got_o, got_l, rep = OB.edited_grid(occ, lab, T, moves, EXT, lv, boxes, 2, pieces, rest)
    o, l = _np(occ, lab)
    want_o, want_l, landed, over = AO.grid_edit(o, l, o, l, T, EXT, _oracle_moves(o, l, lv, moves, pieces, rest, boxes), lv)
    np.testing.assert_array_equal(got_o.cpu().numpy(), want_o)
    np.testing.assert_array_equal(got_l.cpu().numpy(), want_l)
    for i, r in enumerate(rep):
        assert r["landed"] == landed[i]
        assert r["overwritten"] == {int(k): int(over[i, k]) for k in np.nonzero(over[i])[0]}
    return got_o, got_l, rep


# ---- 1. edited_grid against the rule --------------------------------------------------------------------------------------------

def test_edited_grid_equals_the_rule_for_translations_turns_and_scales(nets):
    _, nf, _, _ = nets
    occ, lab = _sweep(nf)
    lv = _level(occ)
    o, l = _np(occ, lab)
    a, b = _labels_by_size(o, l, lv, 2)
    A, bb = OB.grid_affine(T, DIM, EXT)
    ca = A @ _centre(o, l, lv, a) + bb
    for m in (OB._translate(A @ np.array([2.0, -3.0, 1.0])), OB._translate((0.05, -0.1, 0.07)), _turn(90.0, ca), _turn(45.0, ca),
              _turn(20.0, ca), np.asarray(OB.manipulation_transform(ca, "scale", scale=1.2)["transformations"][0]["transformation"])):
        _check_edit(occ, lab, lv, [(a, m)])
    _check_edit(occ, lab, lv, [(a, _turn(90.0, ca)), (b, OB._translate(A @ np.array([0.0, 2.0, 0.0])))])


def test_edited_grid_equals_the_rule_with_pieces_both_rests_and_eight_moves(nets):
    _, nf, _, _ = nets
    occ, lab = _sweep(nf)
    lv = _level(occ)
    o, l = _np(occ, lab)
    labels = _labels_by_size(o, l, lv, 8)
    a = labels[0]
    A, _ = OB.grid_affine(T, DIM, EXT)
    cc = OB.object_components(occ, lab, lv, 26)
    piece = OB.component_region(cc, [OB.largest_components(cc["label"], cc["voxels"])[a]], T, EXT, dilate=0)
    for rest in ("keep", "drop"):
        _check_edit(occ, lab, lv, [(a, OB._translate(A @ np.array([1.0, 2.0, -2.0])))], [piece], rest)
    moves = [(k, OB._translate(A @ np.array([(i % 3) - 1.0, 1.0, (i % 2) * 2.0]))) for i, k in enumerate(labels)]
    _check_edit(occ, lab, lv, moves)


def test_an_empty_box_vacates_and_an_absent_label_and_the_identity_change_nothing(nets):
    _, nf, _, _ = nets
    occ, lab = _sweep(nf)
    lv = _level(occ)
    o, l = _np(occ, lab)
    a = _labels_by_size(o, l, lv, 1)[0]
    absent = next(k for k in range(128) if not (l == k).any())
    A, _ = OB.grid_affine(T, DIM, EXT)
    shift = OB._translate(A @ np.array([2.0, 0.0, 0.0]))
    for moves, boxes in (([(a, shift)], [OB.EMPTY_BOX]), ([(absent, shift)], [(0, DIM - 1) * 3]), ([(a, np.eye(4))], None)):
        got_o, got_l, rep = _check_edit(occ, lab, lv, moves, boxes=boxes)
        assert rep[0]["total"] == 0
        if boxes == [OB.EMPTY_BOX]:                                   # nothing taken, the label's solid points vacated
            assert rep[0]["landed"] == 0 and not ((got_l == a) & (got_o > lv)).any()
        else:
            assert torch.equal(got_o, occ) and torch.equal(got_l, lab)


def test_one_move_reports_what_move_overlap_reports_also_off_the_grid_points(nets):
    _, nf, _, _ = nets
    occ, lab = _sweep(nf)
    lv = _level(occ)
    o, l = _np(occ, lab)
    a = _labels_by_size(o, l, lv, 1)[0]
    A, bb = OB.grid_affine(T, DIM, EXT)
    ca = A @ _centre(o, l, lv, a) + bb
    for m in (OB._translate(A @ np.array([0.0, -2.0, 1.0])), _turn(20.0, ca), OB._translate((0.03, 0.011, -0.07))):
        _, _, rep = OB.edited_grid(occ, lab, T, [(a, m)], EXT, lv)
        ov = OB.move_overlap(occ, lab, T, [(a, m)], EXT, lv)[0]
        assert rep[0]["landed"] == ov["landed"] and rep[0]["overwritten"] == ov["overlap"] and rep[0]["total"] == ov["total"]


def test_edited_grid_equals_edited_sweep_on_the_exact_grid(nets):
    _, nf, _, _ = nets
    occ, lab = _sweep(nf)
    lv = 0.45 if float(occ.min()) < 0.45 < float(occ.max()) else _level(occ)
    o, l = _np(occ, lab)
    labels = _labels_by_size(o, l, lv, 3)
    A, bb = OB.grid_affine(T, DIM, EXT)
    pivot = A @ np.round(_centre(o, l, lv, labels[0])) + bb
    moves = [(labels[0], _turn(90.0, pivot)), (labels[1], OB._translate(A @ np.array([3.0, 0.0, -2.0]))),
             (labels[2], OB._translate(A @ np.array([0.0, -1.0, 0.0])))]
    for n in (1, 3):
        got_o, got_l, _ = OB.edited_grid(occ, lab, T, moves[:n], EXT, lv)
        want_o, want_l = OB.edited_sweep(nf, T, moves[:n], DIM, EXT, lv, NEAR, FAR, NI)
        assert torch.equal(got_o, want_o) and torch.equal(got_l, want_l)


# ---- 2. placement in a scene ------------------------------------------------------------------------------------------------------

def _downs():
    A, _ = OB.grid_affine(T, 2, EXT)
    return [s * A[:, a] for a in range(3) for s in (1, -1)]


def test_in_scene_maps_with_the_scene_the_source_equal_todays_maps(nets):
    _, nf, _, _ = nets
    occ, lab = _sweep(nf)
    lv = _level(occ, 0.95)
    o, l = _np(occ, lab)
    a = _labels_by_size(o, l, lv, 3)[-1]
    m0 = OB.placement_map(occ, lab, T, a, DOWN, 0, EXT, lv)
    m1 = OB.placement_map(occ, lab, T, a, DOWN, 0, EXT, lv, scene=(occ, lab))
    for k in ("drop", "contacts", "support"):
        assert torch.equal(m0[k], m1[k])
    maps0, _, _ = OB.turned_placement_maps(occ, lab, T, a, DOWN, 4, 0, EXT, lv)
    maps1, _, _ = OB.turned_placement_maps(occ, lab, T, a, DOWN, 4, 0, EXT, lv, scene=(occ, lab))
    for (_, x), (_, y) in zip(maps0, maps1):
        assert all(torch.equal(x[k], y[k]) for k in ("drop", "contacts", "support"))
    ok = np.argwhere(m0["drop"].cpu().numpy() >= 0)
    if len(ok):
        u, v = int(ok[0][0]) + m0["offset_lo"][0], int(ok[0][1]) + m0["offset_lo"][1]
        assert OB.placement(m0, u, v)["contacts"] == OB.placement(m1, u, v)["contacts"]


def test_in_scene_maps_equal_the_rule_in_an_edited_scene(nets):
    _, nf, _, _ = nets
    occ, lab = _sweep(nf)
    lv = _level(occ, 0.95)
    o, l = _np(occ, lab)
    big, a = _labels_by_size(o, l, lv, 2)
    A, _ = OB.grid_affine(T, DIM, EXT)
    s_occ, s_lab, _ = OB.edited_grid(occ, lab, T, [(big, OB._translate(A @ np.array([2.0, 3.0, -1.0])))], EXT, lv)
    so, sl = _np(s_occ, s_lab)
    cc = OB.object_components(occ, lab, lv, 26)
    piece = OB.component_region(cc, [OB.largest_components(cc["label"], cc["voxels"])[a]], T, EXT, dilate=0)
    cases = [(d, 0, None, "keep") for d in _downs()] + [(DOWN, 3, None, "keep"), (DOWN, 0, piece, "keep"), (DOWN, 0, piece, "drop")]
    for down, lift, pc, rest in cases:
        try:
            m = OB.placement_map(occ, lab, T, a, down, lift, EXT, lv, pc, rest, scene=(s_occ, s_lab))
        except ValueError:                                           # the top out of the grid at this lift
            continue
        axis, sign = PO.down_axis(T, EXT, down)
        p = None if pc is None else E.Piece(pc.bits.cpu().numpy(), pc.dim, pc.voxel_map, pc.outside == "keep")
        want = AO.placement_in_scene(o, l, so, sl, T, EXT, a, lv, axis, sign, lift, np.eye(4), m["box"], p, rest == "drop")
        for k in ("drop", "contacts", "support"):
            np.testing.assert_array_equal(m[k].cpu().numpy(), want[k], err_msg="%s down %s" % (k, down))
        ok = np.argwhere(want["drop"] >= 0)
        for iu, iv in ok[np.linspace(0, len(ok) - 1, min(4, len(ok))).astype(int)] if len(ok) else []:
            u, v = int(iu) + m["offset_lo"][0], int(iv) + m["offset_lo"][1]
            got = OB.placement(m, u, v)
            assert got["contacts"] == PO.support_cells(want, u, v) and got["stable"] == PO.stable(want, u, v)


# ---- 3. arrange_objects ---------------------------------------------------------------------------------------------------------

def _hand_scene():
    """[i, j, k] with height along +i (down = network -x): a floor (6), a table (1), two boxes (2, 3)."""
    d = 17
    occ, labels = np.zeros((d,) * 3, dtype=np.float32), np.zeros((d,) * 3, dtype=np.int16)
    occ[0], labels[0] = 0.9, 6
    occ[4, 1:6, 1:6], labels[4, 1:6, 1:6] = 0.9, 1
    for j in (1, 5):
        for k in (1, 5):
            occ[1:4, j, k], labels[1:4, j, k] = 0.9, 1
    occ[1:3, 12:14, 12:14], labels[1:3, 12:14, 12:14] = 0.9, 2
    occ[1:4, 8:10, 13:16], labels[1:4, 8:10, 13:16] = 0.9, 3
    return occ, labels


def test_arrangements_on_hand_built_grids_equal_the_rule():
    occ, labels = _hand_scene()
    d = occ.shape[0]
    A, b = OB.grid_affine(T, d, EXT)
    net = lambda *i: A @ np.array(i, dtype=np.float64) + b            # noqa: E731
    g_occ, g_lab = torch.from_numpy(occ).to(DEV), torch.from_numpy(labels).to(DEV)
    cases = [[{"label": 1, "near": net(0, 10, 4)}, {"label": 2, "near": net(0, 10, 4), "on": [1], "lift": 4}],
             [{"label": 2, "near": net(0, 8, 8)}, {"label": 3, "near": net(0, 8, 8), "turns": 4}],
             [{"label": 3, "near": net(0, 3, 3), "on": [5]}, {"label": 2, "near": net(0, 9, 14), "stable": False}]]
    for items in cases:
        r = OB.arrange_objects(g_occ, g_lab, T, items, (-1.0, 0.0, 0.0), EXT, 0.45)
        want_o, want_l, chosen = AO.arrange(occ, labels, T, EXT, items, (-1.0, 0.0, 0.0), 0.45)
        np.testing.assert_array_equal(r["occ"].cpu().numpy(), want_o)
        np.testing.assert_array_equal(r["labels"].cpu().numpy(), want_l)
        for it, c in zip(r["items"], chosen):
            assert (it["placement"] is None) == (c is None)
            if c is not None:
                assert it["placement"]["offset"] == c["offset"] and it["placement"]["drop"] == c["drop"] and it["turn"] == c["turn"]
                np.testing.assert_array_equal(np.asarray(it["placement"]["transformation"]), c["trans"])


def _cube_piece(occ, lab, lv, label):
    """The piece of `label` inside the index cube of side DIM / 4 around its centre: a small object with many offsets."""
    _, _, centre = OB._object_extent((lab == label) & (occ > lv))
    lo = [min(max(int(c) - DIM // 8, 0), DIM - DIM // 4) for c in centre]
    cube = torch.zeros((DIM,) * 3, dtype=torch.bool, device=occ.device)
    cube[lo[0]:lo[0] + DIM // 4, lo[1]:lo[1] + DIM // 4, lo[2]:lo[2] + DIM // 4] = True
    return OB.region_from_mask(cube, T, EXT, applies=[label], outside="drop")


def _arrange_synthetic(nf, turns):
    """4 small pieces (rest dropped, so that each label is its piece after the move) aimed around the grid's centre."""
    occ, lab = _sweep(nf)
    lv = _level(occ, 0.99)
    o, l = _np(occ, lab)
    labels = list(dict.fromkeys(_labels_by_size(o, l, lv, 4)))
    A, b = OB.grid_affine(T, DIM, EXT)
    aims = [A @ np.array([j, DIM // 2, k], dtype=np.float64) + b for j, k in ((8, 8), (8, 24), (24, 8), (24, 24))]
    items = [{"label": k, "near": x, "turns": turns, "stable": False, "piece": _cube_piece(occ, lab, lv, k), "rest": "drop"}
             for k, x in zip(labels, aims)]
    r = OB.arrange_objects(occ, lab, T, items, DOWN, EXT, lv)
    if not r["moves"]:
        pytest.skip("no piece of this synthetic sweep rests on anything at level %g" % lv)
    return occ, lab, lv, items, r


def test_an_arrangement_is_the_grid_edit_of_its_moves_and_overwrites_nothing_at_quarter_turns(nets):
    _, nf, _, _ = nets
    for turns in (4, 8):
        occ, lab, lv, items, r = _arrange_synthetic(nf, turns)
        o2, l2, rep = OB.edited_grid(occ, lab, T, r["moves"], EXT, lv, pieces=r["pieces"], rest=r["rest"])
        assert torch.equal(o2, r["occ"]) and torch.equal(l2, r["labels"])
        o, l = _np(occ, lab)
        for it, rp in zip([x for x in r["items"] if x["placement"] is not None], r["report"]):
            if it["turn"] is None or it["turn"] % 90.0 == 0.0:
                assert rp["total"] == 0, (it["label"], it["turn"], rp)
            else:
                assert rp["total"] <= TO.near_ties(T, EXT, DIM, it["placement"]["transformation"])
        again = OB.arrange_objects(occ, lab, T, items, DOWN, EXT, lv)
        assert torch.equal(again["occ"], r["occ"]) and torch.equal(again["labels"], r["labels"])
        assert [np.asarray(m).tolist() for _, m in again["moves"]] == [np.asarray(m).tolist() for _, m in r["moves"]]


def test_an_arrangement_at_quarter_turns_is_the_edited_sweep_on_the_exact_grid(nets):
    _, nf, _, _ = nets
    occ, lab, lv, items, r = _arrange_synthetic(nf, 4)
    want_o, want_l = OB.edited_sweep(nf, T, r["moves"], DIM, EXT, lv, NEAR, FAR, NI, pieces=r["pieces"], rest=r["rest"])
    assert torch.equal(want_o, r["occ"]) and torch.equal(want_l, r["labels"])
    inv = OB.inventory_from_grid(r["occ"], r["labels"], T, EXT, lv, objects=[k for k, _ in r["moves"]])
    for it in r["items"]:
        if it["placement"] is None:
            continue
        e = next(x for x in inv if x["label"] == it["label"])
        assert np.abs(np.asarray(e["centre"]) - it["placement"]["centre"]).max() < 1e-12


# ---- 4. rejections, repeatability and the tool ------------------------------------------------------------------------------------

def _call_grid_edit(src, state, moves, dim=DIM):
    ctx = get_context(torch.device(DEV))
    n = max(len(moves), 1)
    landed, over = np.zeros(n, dtype=np.int64), np.zeros((n, 128), dtype=np.int64)
    descs = (_lib.EditMove * n)()
    for i, (k, m) in enumerate(moves):
        descs[i].label = k
        descs[i].trans[:] = np.asarray(m, dtype=np.float64)[:3].reshape(-1).tolist()
        descs[i].box[:] = [0, dim - 1] * 3
    ctx.call("dmnerf_grid_edit", ctx.handle, _lib.ptr(src[0]), _lib.ptr(src[1], torch.int16), dim, 0.45, _lib.doubles(T, 16),
             _lib.doubles(EXT, 3), descs, len(moves), _lib.ptr(state[0]), _lib.ptr(state[1], torch.int16),
             landed.ctypes.data_as(C.POINTER(C.c_int64)), over.ctypes.data_as(C.POINTER(C.c_int64)))


def test_the_library_rejects_bad_calls_and_leaves_the_state_unwritten():
    occ = torch.full((DIM,) * 3, 0.9, device=DEV)
    lab = torch.ones((DIM,) * 3, dtype=torch.int16, device=DEV)
    state = (occ.clone(), lab.clone())
    shift = OB._translate((0.25, 0.0, 0.0))
    with pytest.raises(RuntimeError, match="overlap in memory"):
        _call_grid_edit((occ, lab), (occ, lab), [(1, shift)])
    for moves in ([], [(1, shift)] * 9, [(128, shift)], [(1, np.diag([1.0, 1.0, -1.0, 1.0]))]):
        with pytest.raises(RuntimeError):
            _call_grid_edit((occ, lab), state, moves)
    for bad in ("src", "state"):
        s_occ, st = occ.clone(), (state[0].clone(), state[1].clone())
        (s_occ if bad == "src" else st[0])[3, 4, 5] = float("nan")
        before = (st[0].clone(), st[1].clone())
        with pytest.raises(RuntimeError, match="NaN"):
            _call_grid_edit((s_occ, lab), st, [(1, shift)])
        assert torch.equal(torch.nan_to_num(st[0]), torch.nan_to_num(before[0])) and torch.equal(st[1], before[1])
    with pytest.raises(ValueError):
        OB.placement_map(occ, lab, T, 1, DOWN, 0, EXT, scene=(occ[:-1], lab))
    with pytest.raises(ValueError):
        OB.edited_grid(occ, lab, T, [(1, shift)] * 9, EXT)


def test_move_objects_arrange_writes_what_the_library_returns(nets, tmp_path):
    nc, nf, _, _ = nets
    ck = tmp_path / "ck.tar"
    torch.save({"network_coarse_state_dict": {k: v.cpu() for k, v in nc.state_dict().items()},
                "network_fine_state_dict": {k: v.cpu() for k, v in nf.state_dict().items()}}, str(ck))
    np.save(str(tmp_path / "pose.npy"), np.eye(4, dtype=np.float32)[:3])
    np.save(str(tmp_path / "T.npy"), T)
    occ, lab = _sweep(nf)
    lv = _level(occ)
    o, l = _np(occ, lab)
    ins_num = int(nf.ins_linear.weight.shape[0]) - 1
    labels = sorted({k for k in _labels_by_size(o, l, lv, 6) if k != ins_num})[:2]
    A, b = OB.grid_affine(T, DIM, EXT)
    spec = [{"label": k, "near": (A @ np.array([16.0, j, 16.0]) + b).tolist(), "turns": 2, "any_stability": True}
            for k, j in zip(labels, (8.0, 24.0))]
    (tmp_path / "spec.json").write_text(json.dumps(spec))
    out = tmp_path / "out"
    cmd = [sys.executable, os.path.join(ROOT, "tools", "move_objects.py"), str(ck), "--pose", str(tmp_path / "pose.npy"), "--hwk", "8",
           "8", "10", "0", "4", "0", "10", "4", "0", "0", "1", "--transform", str(tmp_path / "T.npy"), "--extents", "4", "4", "4",
           "--grid-dim", str(DIM), "--level", str(lv), "--arrange", str(tmp_path / "spec.json"), "--down", *map(str, DOWN),
           "--dilate", "0", "--out", str(out), "--N-test", "64"]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    rec = json.loads(open(out / "transform.json").read())
    assert len(rec["arrange"]) == len(spec) and os.path.exists(out / "rgb.png")
    placed = [e for e in rec["arrange"] if e["placed"]]
    assert len(placed) == len(rec["transformations"]) and rec["labels"] == [e["label"] for e in placed]
    for e in placed:
        assert "overwritten" in e and len(e["offset"]) == 2 and e["turn"] in (0.0, 180.0)
