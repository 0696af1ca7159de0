"""GPU: turned placements -- dmnerf_placement_maps and dmnerf_placement_contacts_moved against the numpy rule
(oracle/placement_turn_oracle.py) on synthetic keep-all sweeps and hand-built grids, the identity base against
dmnerf_placement_map, the agreement with the collision checks and the edited sweep, batching, the rejections and the tools'
--turns."""
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
from oracle import edit_sweep_oracle as E
from oracle import placement_oracle as PO
from oracle import placement_turn_oracle as TO

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
NEAR, FAR, NI = 4.0, 15.0, 128
T, DIM, EXT = np.eye(4), 33, (4.0, 4.0, 4.0)       # grid points and 0.125 steps are exact in fp32
QUARTER, OTHER = (0.0, 90.0, 180.0, 270.0), (45.0, 20.0)


@pytest.fixture(scope="module", params=[13, 93])
def nets(request):
    return make_models(101, 202, request.param, DEV)


def _sweep(nf, dim=DIM):
    ins_num = int(nf.ins_linear.weight.shape[0]) - 1
    return OB.occupancy_objects(nf, T, OB.object_mask(ins_num, remove=[]), dim, EXT, NEAR, FAR, NI, device=DEV)


def _level(occ, q=0.85):
    x = occ.flatten().float()
    x = x[x > 0]
    return float(x.kthvalue(max(1, int(q * x.numel()))).values)


def _np(*ts):
    return [t.cpu().numpy() for t in ts]


def _small_label(o, l, lv):
    """The label with the most solid points among those whose horizontal boxes span at most half the grid (else the largest)."""
    k, c = np.unique(l[o > np.float32(lv)], return_counts=True)
    for x in k[np.argsort(-c, kind="stable")]:
        box = E.solid_box(o, l, int(x), lv, 0)
        if max(box[3] - box[2], box[5] - box[4], box[1] - box[0]) < o.shape[0] // 2 and (l == x).sum() > 20:
            return int(x)
    return int(k[np.argmax(c)])


def _downs():
    A, _ = OB.grid_affine(T, 2, EXT)
    return [s * A[:, a] for a in range(3) for s in (1, -1)]


def _oracle_piece(p):
    return None if p is None else E.Piece(p.bits.cpu().numpy(), p.dim, p.voxel_map, p.outside == "keep")


def _scene(rng, dim):
    """[h1, h2, y] with y up: a floor, random blocks of labels 2..9, and object 1: an L-shaped plate with a post below."""
    g = np.zeros((dim,) * 3, dtype=np.float32)
    lab = np.zeros((dim,) * 3, dtype=np.int16)
    g[:, :, 0:2], lab[:, :, 0:2] = 0.9, 10
    for _ in range(40):
        a, b, c = rng.integers(0, dim - 4, 3)
        g[a:a + 4, b:b + 3, c:c + 2], lab[a:a + 4, b:b + 3, c:c + 2] = 0.9, rng.integers(2, 10)
    g[10:16, 8:10, 20:22], lab[10:16, 8:10, 20:22] = 0.9, 1
    g[10:12, 10:14, 20:22], lab[10:12, 10:14, 20:22] = 0.9, 1
    g[12, 9, 15:20], lab[12, 9, 15:20] = 0.9, 1
    return g, lab


def _posed(G, axis, sign):
    g = G[:, :, ::-1] if sign > 0 else G
    h = [a for a in range(3) if a != axis]
    order = [0, 0, 0]
    order[h[0]], order[h[1]], order[axis] = 0, 1, 2
    return np.ascontiguousarray(np.transpose(g, order))


def _check_turns(occ, lab, lv, label, down, angles, lift=0, piece=None, rest="keep", obstacles=None, n_cells=6):
    """Every turn's map and a sample of its placements against the oracle -> [(angle, map)]."""
    o, l = _np(occ, lab)
    maps, unfit, unplaced = OB.turned_placement_maps(occ, lab, T, label, down, angles, lift, EXT, lv, piece, rest, obstacles)
    assert len(maps) + len(unfit) + len(unplaced) == len(angles)
    axis, sign = PO.down_axis(T, EXT, down)
    for angle, m in maps:
        assert m["base"] is not None and (m["axis"], m["sign"]) == (axis, sign)
        want = TO.placement_map(o, l, T, EXT, label, lv, axis, sign, lift, m["base"], m["box"], _oracle_piece(piece), rest == "drop",
                                obstacles)
        for k in ("drop", "contacts", "support"):
            np.testing.assert_array_equal(m[k].cpu().numpy(), want[k], err_msg="%s at %g degrees" % (k, angle))
        assert m["offset_lo"] == want["offset_lo"] and m["points"] == want["points"].shape[0]
        h = m["horizontal"]
        assert [m["centre"][h[0]], m["centre"][h[1]]] == want["centre"][:2]
        ok = np.argwhere(want["drop"] >= 0)
        for iu, iv in ok[np.linspace(0, len(ok) - 1, min(n_cells, len(ok))).astype(int)] if len(ok) else []:
            u, v = int(iu) + m["offset_lo"][0], int(iv) + m["offset_lo"][1]
            p = OB.placement(m, u, v)
            assert p["contacts"] == PO.support_cells(want, u, v) and p["stable"] == PO.stable(want, u, v)
            assert p["drop"] == want["drop"][iu, iv]
    return maps


# ---- 1. against the numpy rule ------------------------------------------------------------------------------------------------

def test_turned_maps_equal_the_rule_in_all_six_directions(nets):
    _, nf, _, _ = nets
    occ, lab = _sweep(nf)
    lv = _level(occ, 0.95)
    o, l = _np(occ, lab)
    label = _small_label(o, l, lv)
    mapped = 0
    for down in _downs():
        mapped += len(_check_turns(occ, lab, lv, label, down, QUARTER[1:] + OTHER))
    assert mapped
    _check_turns(occ, lab, lv, label, (0, -1, 0), (90.0, 45.0), lift=3)


def test_pieces_rest_policies_and_obstacle_masks_equal_the_rule(nets):
    _, nf, _, _ = nets
    occ, lab = _sweep(nf)
    lv = _level(occ, 0.95)
    o, l = _np(occ, lab)
    label = _small_label(o, l, lv)
    cc = OB.object_components(occ, lab, lv, 26)
    piece = OB.component_region(cc, [OB.largest_components(cc["label"], cc["voxels"])[label]], T, EXT, dilate=0)
    for rest in ("keep", "drop"):
        _check_turns(occ, lab, lv, label, (0, -1, 0), (90.0, 20.0), 0, piece, rest)
    _check_turns(occ, lab, lv, label, (1, 0, 0), (270.0, 45.0), 2, obstacles=[k for k in range(128) if k % 2])


def test_hand_built_grids_equal_the_rule_in_all_six_directions():
    G, L = _scene(np.random.default_rng(2), DIM)
    A, _ = OB.grid_affine(T, DIM, EXT)
    for axis in range(3):
        for sign in (1, -1):
            occ, lab = torch.from_numpy(_posed(G, axis, sign)).to(DEV), torch.from_numpy(_posed(L, axis, sign)).to(DEV)
            maps = _check_turns(occ, lab, 0.45, 1, sign * A[:, axis], QUARTER + OTHER, lift=2, n_cells=10)
            assert len(maps) == 6
            drops = [m["drop"].cpu().numpy() for _, m in maps]
            assert any((d >= 0).any() and (d < 0).any() for d in drops)


# ---- 2. the identity, the collision checks, the edit and batching -------------------------------------------------------------

def test_the_identity_base_equals_the_unmoved_map_bit_for_bit(nets):
    _, nf, _, _ = nets
    occ, lab = _sweep(nf)
    for q in (0.85, 0.95):
        lv = _level(occ, q)
        o, l = _np(occ, lab)
        label = _small_label(o, l, lv)
        for down in _downs():
            m0 = OB.placement_map(occ, lab, T, label, down, 0, EXT, lv)
            m1 = OB.placement_map(occ, lab, T, label, down, 0, EXT, lv, base=np.eye(4))
            for k in ("drop", "contacts", "support"):
                assert torch.equal(m0[k], m1[k]), k
            for k in ("offset_lo", "centre", "runs", "points", "height"):
                assert m0[k] == m1[k], k
            assert m1["points_before"] == m1["points"]


def _collisions(occ, lab, lv, label, m, exact):
    """Every resting offset's move (a sample of 64 when not exact) against move_overlap -> the largest near-tie count."""
    drop, support = m["drop"].cpu().numpy(), m["support"].cpu().numpy()
    A, _ = OB.grid_affine(T, DIM, EXT)
    ok = np.argwhere(drop >= 0)
    if not exact:
        ok = ok[np.linspace(0, len(ok) - 1, min(64, len(ok))).astype(int)] if len(ok) else ok
    moves, lower = [], []
    for iu, iv in ok:
        u, v = iu + m["offset_lo"][0], iv + m["offset_lo"][1]
        moves.append(m["base"] @ OB.placement_transform(A, OB.placement_delta(m, u, v, drop[iu, iv])))
        lower.append(m["base"] @ OB.placement_transform(A, OB.placement_delta(m, u, v, drop[iu, iv] + 1)))
    ties = 0
    for s in range(0, len(moves), _lib.MAX_CANDIDATES // 2):
        mv, lw = moves[s:s + _lib.MAX_CANDIDATES // 2], lower[s:s + _lib.MAX_CANDIDATES // 2]
        r = OB.move_overlap(occ, lab, T, [(label, t) for t in mv + lw], EXT, lv, [m["box"]] * 2 * len(mv))
        for i, x in enumerate(r[:len(mv)]):
            if exact:
                assert x["total"] == 0 and x["landed"] == m["points"]
            else:
                n = max(TO.near_ties(T, EXT, DIM, mv[i]), TO.near_ties(T, EXT, DIM, m["base"]))
                ties = max(ties, n)
                assert x["total"] <= n and abs(x["landed"] - m["points"]) <= n
        if exact:
            sup = support[ok[s:s + len(mv), 0], ok[s:s + len(mv), 1]] >= 0
            assert all(x["total"] > 0 for x, s_ in zip(r[len(mv):], sup) if s_)
    return ties


def test_turned_objects_land_as_the_collision_checks_see_them(nets, capsys):
    _, nf, _, _ = nets
    occ, lab = _sweep(nf)
    lv = _level(occ, 0.95)
    o, l = _np(occ, lab)
    label = _small_label(o, l, lv)
    seen = 0
    ties = 0
    for down in ((0, -1, 0), (-1, 0, 0), (0, 0, 1)):
        maps, _, _ = OB.turned_placement_maps(occ, lab, T, label, down, QUARTER + OTHER, 0, EXT, lv)
        for angle, m in maps:
            r = OB.move_overlap(occ, lab, T, [(label, m["base"])], EXT, lv, [m["box"]])[0]
            assert r["landed"] == m["points"]                                # |S_base| is move_overlap(base).landed
            if (m["drop"] >= 0).any():
                ties = max(ties, _collisions(occ, lab, lv, label, m, angle in QUARTER))
                seen += 1
    assert seen
    with capsys.disabled():
        print("\nturned placements: at most %d near-tie points at the non-quarter angles %s" % (ties, OTHER))


def test_place_object_with_turns_through_edited_sweep_lands_on_nothing(nets):
    _, nf, _, _ = nets
    occ, lab = _sweep(nf)
    o, l = _np(occ, lab)
    A, b = OB.grid_affine(T, DIM, EXT)
    near = A @ np.full(3, (DIM - 1) / 2.0) + b
    found = 0
    cases = []
    for lv in (_level(occ, q) for q in (0.85, 0.95, 0.99)):
        k, c = np.unique(l[o > np.float32(lv)], return_counts=True)
        cases += [(lv, int(x), d) for x in k[np.argsort(-c, kind="stable")] for d in _downs()]
    for lv, label, down in cases:
        if found == 3:
            break
        r = OB.place_object(occ, lab, T, label, down, near, stable=False, extents=EXT, level=lv, turns=4)
        p = r["placement"]
        assert len(r["maps"]) + len(r["unfit"]) + len(r["unplaced"]) == 4
        if p is None:
            assert r["candidates"] == 0 and r["reason"] and r["turn"] is None
            continue
        found += 1
        assert r["turn"] in QUARTER and r["tested"] == 1 and p["supported"]
        eo, el = _np(*OB.edited_sweep(nf, T, [(label, p["transformation"])], DIM, EXT, lv, NEAR, FAR, NI))
        over = (o > lv) & (l != label) & (el == label) & (eo > lv)
        assert not over.any()
        e = OB.inventory_from_grid(torch.from_numpy(eo).to(DEV), torch.from_numpy(el).to(DEV), T, EXT, lv, objects=[label])[0]
        np.testing.assert_allclose(e["centre"], p["centre"], rtol=0, atol=1e-12)
    assert found or len(np.unique(l[o > np.float32(_level(occ))])) == 1


def test_a_batched_call_equals_one_call_per_base_and_repeats_bit_for_bit(nets):
    _, nf, _, _ = nets
    occ, lab = _sweep(nf)
    lv = _level(occ, 0.95)
    o, l = _np(occ, lab)
    label = _small_label(o, l, lv)
    angles = [360.0 * k / 36 for k in range(36)]
    maps, unfit, _ = OB.turned_placement_maps(occ, lab, T, label, (0, -1, 0), angles, 0, EXT, lv)
    again, _, _ = OB.turned_placement_maps(occ, lab, T, label, (0, -1, 0), angles, 0, EXT, lv)
    assert [a for a, _ in maps] == [a for a, _ in again] and len(maps) + len(unfit) == 36
    for (angle, m), (_, m2) in zip(maps, again):
        one = OB.placement_map(occ, lab, T, label, (0, -1, 0), 0, EXT, lv, base=m["base"], box=m["box"])
        for k in ("drop", "contacts", "support"):
            assert torch.equal(m[k], one[k]) and torch.equal(m[k], m2[k]), (k, angle)
        assert m["centre"] == one["centre"] and m["offset_lo"] == one["offset_lo"] and m["points"] == one["points"]


# ---- 3. rejections and statuses ----------------------------------------------------------------------------------------------

def test_the_library_rejects_bad_input_and_reports_unplaced_bases():
    dim = 8
    occ = torch.zeros((dim,) * 3, device=DEV)
    lab = torch.zeros((dim,) * 3, device=DEV, dtype=torch.int16)
    occ[2:4, 2:4, 2:4], lab[2:4, 2:4, 2:4] = 0.9, 1
    ctx = get_context(DEV)
    eye = np.eye(4)[:3].reshape(-1)
    whole = (0, dim - 1) * 3

    def maps(bases, box=whole, n=None, lift=0):
        desc = _lib.Placement(label=1, axis=0, sign=-1, lift=lift)
        desc.obstacles[:] = OB.ALL_LABELS
        rows = np.ascontiguousarray(np.asarray(bases, dtype=np.float64).reshape(-1, 12))
        n = rows.shape[0] if n is None else n
        k = max(n, 1)
        out = [torch.zeros(k * dim * dim, dtype=t, device=DEV) for t in (torch.int32, torch.int32, torch.int16)]
        infos = (_lib.PlacementInfo * k)()
        status = np.full(k, -7, dtype=np.int32)
        ctx.call("dmnerf_placement_maps", ctx.handle, _lib.ptr(occ), _lib.ptr(lab, torch.int16), dim, 0.45, _lib.doubles(np.eye(4), 16),
                 _lib.doubles((4.0, 4.0, 4.0), 3), C.byref(desc), rows.ctypes.data_as(C.POINTER(C.c_double)), (C.c_int32 * 6)(*box), n,
                 _lib.ptr(out[0], torch.int32), _lib.ptr(out[1], torch.int32), _lib.ptr(out[2], torch.int16), infos,
                 status.ctypes.data_as(C.POINTER(C.c_int32)))
        return status, infos, out

    def rejected(*a, **kw):
        with pytest.raises(RuntimeError) as e:
            maps(*a, **kw)
        return str(e.value)

    assert "between 1 and 64" in rejected([eye], n=0) and "between 1 and 64" in rejected([eye] * 65)
    nan = eye.copy()
    nan[3] = np.nan
    flip = np.diag([1.0, 1.0, -1.0])
    bad = np.concatenate([flip, np.zeros((3, 1))], 1).reshape(-1)
    assert "not finite" in rejected([eye, nan]) and "det" in rejected([bad])
    assert "inverted" in rejected([eye], box=(3, 2, 0, 7, 0, 7)) and "outside the grid" in rejected([eye], box=(0, dim) * 3)
    far = eye.copy()
    far[3] = 100.0                                                   # everything is sampled outside the grid: no point
    status, infos, out = maps([eye, far, eye])
    assert status.tolist() == [0, 1, 0] and infos[1].points == 0 and infos[0].points == infos[2].points == 8
    for t in out:
        assert torch.equal(t[:dim * dim], t[2 * dim * dim:])
    status, _, _ = maps([eye], lift=5)
    assert status.tolist() == [2]
    with pytest.raises(ValueError, match="after the move"):
        OB.placement_map(occ, lab, np.eye(4), 1, (-1, 0, 0), extents=(4.0, 4.0, 4.0), base=OB._translate((100.0, 0, 0)))
    m = OB.placement_map(occ, lab, np.eye(4), 1, (-1, 0, 0), extents=(4.0, 4.0, 4.0), base=np.eye(4))
    with pytest.raises(ValueError, match="outside"):
        OB.placement(m, 7, 0)
    desc = _lib.Placement(label=1, axis=0, sign=-1, lift=0)
    desc.obstacles[:] = OB.ALL_LABELS
    cells, n, dr = np.zeros((8, 3), dtype=np.int32), C.c_int64(0), C.c_int32(0)
    for base, msg in ((far, "after the move"), (nan, "not finite")):
        with pytest.raises(RuntimeError, match=msg):
            ctx.call("dmnerf_placement_contacts_moved", ctx.handle, _lib.ptr(occ), _lib.ptr(lab, torch.int16), dim, 0.45,
                     _lib.doubles(np.eye(4), 16), _lib.doubles((4.0, 4.0, 4.0), 3), C.byref(desc), _lib.doubles(base, 12),
                     (C.c_int32 * 6)(*whole), 0, 0, cells.ctypes.data_as(C.POINTER(C.c_int32)), 8, C.byref(n), C.byref(dr))


# ---- 4. tools ----------------------------------------------------------------------------------------------------------------

def test_move_objects_and_find_objects_with_turns_write_what_the_library_returns(tmp_path):
    nc, nf, _, _ = make_models(7, 8, 13, "cpu", trained_like=True)
    torch.save({"network_coarse_state_dict": nc.state_dict(), "network_fine_state_dict": nf.state_dict()}, tmp_path / "ck.tar")
    np.save(tmp_path / "T.npy", np.eye(4))
    nf = make_models(7, 8, 13, DEV, trained_like=True)[1]
    pose = np.eye(4, dtype=np.float32)
    pose[2, 3] = 6.0
    np.save(tmp_path / "pose.npy", pose)
    ext = (1.9, 7.0, 7.0)
    o, l = _np(*OB.occupancy_objects(nf, np.eye(4), OB.object_mask(13, keep=range(13)), 32, ext, device=DEV))
    lv = _level(torch.from_numpy(o), 0.5)
    label = _small_label(o, l, lv)
    near = [0.0, 0.5, 0.0]
    argv = [str(tmp_path / "ck.tar"), "--pose", str(tmp_path / "pose.npy"), "--hwk", "24", "32", "30", "0", "16", "0", "30", "12", "0",
            "0", "1", "--move-label", str(label), "--transform", str(tmp_path / "T.npy"), "--grid-dim", "32", "--level", repr(lv),
            "--out", str(tmp_path / "o"), "--N-test", "256", "--place-at"] + [repr(x) for x in near] + \
        ["--down", "0", "-1", "0", "--any-stability", "--turns", "4"]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "move_objects.py")] + argv, capture_output=True, text=True)
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import move_objects
    a = move_objects.parse(argv)
    _, lab_, _, region = move_objects.choose_piece(a, nf, np.eye(4), ext)
    occ, lab = OB.occupancy_objects(nf, np.eye(4), OB.object_mask(13, remove=[]), 32, ext, device=DEV)
    want = OB.place_object(occ, lab, np.eye(4), lab_, (0, -1, 0), near, stable=False, extents=ext, level=lv, piece=region, turns=4)
    if want["placement"] is None:
        assert r.returncode != 0 and "no placement" in r.stderr
    else:
        assert r.returncode == 0, r.stderr[-3000:]
        info = json.loads(r.stdout.strip().splitlines()[-1])
        p = want["placement"]
        assert info["place"] == {"offset": list(p["offset"]), "drop": p["drop"], "support": p["support"], "stable": p["stable"],
                                 "contacts": [list(c) for c in p["contacts"]], "turn": want["turn"]}
        assert info["transformations"][0]["transformation"] == p["transformation"]
    base = [sys.executable, os.path.join(ROOT, "tools", "find_objects.py"), str(tmp_path / "ck.tar"), "--transform",
            str(tmp_path / "T.npy"), "--grid-dim", "32", "--level", repr(lv), "--out", str(tmp_path / "f")]
    r = subprocess.run(base + ["--placements", str(label), "--down", "0", "-1", "0", "--turns", "4"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    info = json.loads(r.stdout.strip().splitlines()[-1])
    z = np.load(tmp_path / "f" / info["placements"])
    maps, unfit, unplaced = OB.turned_placement_maps(occ, lab, np.eye(4), label, (0, -1, 0), 4, 0, ext, lv)
    assert z["angles"].tolist() == [a_ for a_, _ in maps] and z["unfit"].tolist() == unfit
    for t, (_, m) in enumerate(maps):
        for k in ("drop", "support", "contacts"):
            np.testing.assert_array_equal(z["%s_%d" % (k, t)], m[k].cpu().numpy())
        assert tuple(z["offset_lo_%d" % t]) == m["offset_lo"]
        np.testing.assert_array_equal(z["base_%d" % t], m["base"])
