"""GPU: object placement -- dmnerf_placement_map and dmnerf_placement_contacts against the brute-force numpy rule
(oracle/placement_oracle.py) on synthetic keep-all sweeps and on hand-built grids, the agreement with the collision checks and
the edited sweep, the rejections and the tools' --place-at / --placements."""
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

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
NEAR, FAR, NI = 4.0, 15.0, 128
T, DIM, EXT = np.eye(4), 33, (4.0, 4.0, 4.0)       # grid points and 0.125 steps are exact in fp32


@pytest.fixture(scope="module", params=[13, 93])
def nets(request):
    return make_models(101, 202, request.param, DEV)


def _sweep(nf, dim=DIM, T_=T, ext=EXT):
    ins_num = int(nf.ins_linear.weight.shape[0]) - 1
    return OB.occupancy_objects(nf, T_, OB.object_mask(ins_num, remove=[]), dim, ext, NEAR, FAR, NI, device=DEV)


def _level(occ, q=0.85):
    x = occ.flatten().float()
    x = x[x > 0]
    lv = float(x.kthvalue(max(1, int(q * x.numel()))).values)
    assert 0.0 < lv < 1.0
    return lv


def _np(*ts):
    return [t.cpu().numpy() for t in ts]


def _top_label(o, l, lv):
    k, c = np.unique(l[o > np.float32(lv)], return_counts=True)
    return int(k[np.argmax(c)])


def _downs(T_, ext):
    A, _ = OB.grid_affine(T_, 2, ext)
    return [s * A[:, a] for a in range(3) for s in (1, -1)]


def _oracle_piece(p):
    return None if p is None else E.Piece(p.bits.cpu().numpy(), p.dim, p.voxel_map, p.outside == "keep")


def _check_map(occ, lab, T_, ext, lv, label, down, lift, piece=None, rest="keep", obstacles=None, n_cells=12):
    """The map and a sample of placements against the oracle -> (map, oracle map)."""
    o, l = _np(occ, lab)
    m = OB.placement_map(occ, lab, T_, label, down, lift, ext, lv, piece, rest, obstacles)
    axis, sign = PO.down_axis(T_, ext, down)
    assert (m["axis"], m["sign"]) == (axis, sign)
    want = PO.placement_map(o, l, T_, ext, label, lv, axis, sign, lift, _oracle_piece(piece), rest == "drop", obstacles)
    for k in ("drop", "contacts", "support"):
        np.testing.assert_array_equal(m[k].cpu().numpy(), want[k], err_msg=k)
    assert m["offset_lo"] == want["offset_lo"] and m["points"] == want["points"].shape[0]
    h = m["horizontal"]
    assert [m["centre"][h[0]], m["centre"][h[1]]] == want["centre"][:2]
    ok = np.argwhere(want["drop"] >= 0)
    for iu, iv in ok[np.linspace(0, len(ok) - 1, min(n_cells, len(ok))).astype(int)] if len(ok) else []:
        u, v = int(iu) + m["offset_lo"][0], int(iv) + m["offset_lo"][1]
        p = OB.placement(m, u, v)
        assert p["contacts"] == PO.support_cells(want, u, v) and p["stable"] == PO.stable(want, u, v)
        assert p["drop"] == want["drop"][iu, iv] and p["supported"] == (want["support"][iu, iv] >= 0)
    return m, want


# ---- 1. against the numpy rule ------------------------------------------------------------------------------------------------

def test_synthetic_sweeps_equal_the_rule_in_all_six_directions(nets):
    _, nf, _, _ = nets
    occ, lab = _sweep(nf)
    lv = _level(occ)
    o, l = _np(occ, lab)
    label = _top_label(o, l, lv)
    for down in _downs(T, EXT):
        for lift in (0, 3):
            try:
                _check_map(occ, lab, T, EXT, lv, label, down, lift)
            except ValueError as e:
                assert "out of the grid" in str(e) and lift > 0
    m1 = OB.placement_map(occ, lab, T, label, (0, -1, 0), 0, EXT, lv)
    m2 = OB.placement_map(occ, lab, T, label, (0, -1, 0), 0, EXT, lv)
    for k in ("drop", "contacts", "support"):                                         # bit-reproducible
        assert torch.equal(m1[k], m2[k])


def test_pieces_rest_policies_and_obstacle_masks_equal_the_rule(nets):
    _, nf, _, _ = nets
    occ, lab = _sweep(nf)
    lv = _level(occ)
    o, l = _np(occ, lab)
    label = _top_label(o, l, lv)
    cc = OB.object_components(occ, lab, lv, 26)
    piece = OB.component_region(cc, [OB.largest_components(cc["label"], cc["voxels"])[label]], T, EXT, dilate=0)
    for rest in ("keep", "drop"):
        _check_map(occ, lab, T, EXT, lv, label, (0, -1, 0), 0, piece, rest)
        _check_map(occ, lab, T, EXT, lv, label, (1, 0, 0), 2, piece, rest)
    _check_map(occ, lab, T, EXT, lv, label, (0, 0, -1), 0, obstacles=[k for k in range(128) if k % 2])


def _scene(rng, dim):
    """[h1, h2, y] with y up: a floor, random blocks of labels 2..9 at every height, and object 1: a plate with a post below."""
    g = np.zeros((dim,) * 3, dtype=np.float32)
    lab = np.zeros((dim,) * 3, dtype=np.int16)
    g[:, :, 0:2], lab[:, :, 0:2] = 0.9, 10
    for _ in range(40):
        a, b, c = rng.integers(0, dim - 4, 3)
        g[a:a + 4, b:b + 3, c:c + 2], lab[a:a + 4, b:b + 3, c:c + 2] = 0.9, rng.integers(2, 10)
    g[10:16, 8:12, 20:22], lab[10:16, 8:12, 20:22] = 0.9, 1
    g[12, 9, 15:20], lab[12, 9, 15:20] = 0.9, 1
    g[15, 11, 24:26], lab[15, 11, 24:26] = 0.9, 1                          # a second run above a gap
    return g, lab


def _posed(G, axis, sign):
    g = G[:, :, ::-1] if sign > 0 else G
    h = [a for a in range(3) if a != axis]
    order = [0, 0, 0]
    order[h[0]], order[h[1]], order[axis] = 0, 1, 2
    return np.ascontiguousarray(np.transpose(g, order))


def test_hand_built_grids_equal_the_rule_and_agree_across_directions():
    G, L = _scene(np.random.default_rng(2), 40)
    A, _ = OB.grid_affine(T, 40, EXT)
    ref = {}
    for axis in range(3):
        for sign in (1, -1):
            occ = torch.from_numpy(_posed(G, axis, sign)).to(DEV)
            lab = torch.from_numpy(_posed(L, axis, sign)).to(DEV)
            for lift in (0, 5):
                m, _ = _check_map(occ, lab, T, EXT, 0.45, 1, sign * A[:, axis], lift, n_cells=20)
                got = [m[k].cpu().numpy() for k in ("drop", "contacts", "support")]
                if lift in ref:
                    for a_, b_ in zip(got, ref[lift]):
                        np.testing.assert_array_equal(a_, b_)
                ref.setdefault(lift, got)
    drop, _, support = ref[0]
    assert (drop < 0).any() and (support > 1).any() and len(set(support[support >= 0].tolist())) > 2


# ---- 2. agreement with the collision check and the edit -----------------------------------------------------------------------

def _agreement(occ, lab, T_, ext, lv, label, down, lift, piece=None, rest="keep"):
    m = OB.placement_map(occ, lab, T_, label, down, lift, ext, lv, piece, rest)
    drop, support = m["drop"].cpu().numpy(), m["support"].cpu().numpy()
    A, _ = OB.grid_affine(T_, m["dim"], ext)
    pieces = None if piece is None else [piece]
    box = OB.edit_boxes(occ, lab, [(label, np.eye(4))], T_, ext, lv, 2, pieces)[0]
    ok = np.argwhere(drop >= 0)
    assert len(ok)
    for s in range(0, len(ok), _lib.MAX_CANDIDATES // 2):
        chunk = ok[s:s + _lib.MAX_CANDIDATES // 2]
        moves, lower = [], []
        for iu, iv in chunk:
            u, v = iu + m["offset_lo"][0], iv + m["offset_lo"][1]
            moves.append((label, OB.placement_transform(A, OB.placement_delta(m, u, v, drop[iu, iv]))))
            lower.append((label, OB.placement_transform(A, OB.placement_delta(m, u, v, drop[iu, iv] + 1))))
        n = len(moves)
        r = OB.move_overlap(occ, lab, T_, moves + lower, ext, lv, [box] * 2 * n, 2, None if piece is None else [piece] * 2 * n, rest)
        assert all(x["total"] == 0 for x in r[:n])
        sup = support[chunk[:, 0], chunk[:, 1]] >= 0
        assert all(x["total"] > 0 for x, s_ in zip(r[n:], sup) if s_)
    return m


def test_every_resting_offset_overlaps_nothing_and_one_voxel_lower_overlaps(nets):
    _, nf, _, _ = nets
    occ, lab = _sweep(nf)
    lv = _level(occ)
    o, l = _np(occ, lab)
    label = _top_label(o, l, lv)
    for down, lift in (((0, -1, 0), 0), ((-1, 0, 0), 0), ((0, 0, 1), 0)):
        _agreement(occ, lab, T, EXT, lv, label, down, lift)
    cc = OB.object_components(occ, lab, lv, 26)
    piece = OB.component_region(cc, [OB.largest_components(cc["label"], cc["voxels"])[label]], T, EXT, dilate=0)
    _agreement(occ, lab, T, EXT, lv, label, (0, -1, 0), 0, piece, "keep")
    G, L = _scene(np.random.default_rng(4), 40)
    A, _ = OB.grid_affine(T, 40, EXT)
    occ2 = torch.from_numpy(_posed(G, 1, -1)).to(DEV)
    lab2 = torch.from_numpy(_posed(L, 1, -1)).to(DEV)
    m = _agreement(occ2, lab2, T, EXT, 0.45, 1, -A[:, 1], 3)
    assert (m["support"] >= 0).any()


def test_slide_until_contact_along_down_finds_the_drop(nets):
    _, nf, _, _ = nets
    occ, lab = _sweep(nf)
    lv = _level(occ)
    o, l = _np(occ, lab)
    label = _top_label(o, l, lv)
    step = EXT[0] / (DIM - 1)
    seen = 0
    for down in _downs(T, EXT):
        m = OB.placement_map(occ, lab, T, label, down, 0, EXT, lv)
        iu, iv = -m["offset_lo"][0], -m["offset_lo"][1]
        drop, support = int(m["drop"][iu, iv]), int(m["support"][iu, iv])
        assert drop >= 0
        r = OB.slide_until_contact(occ, lab, T, label, down, (DIM - 1) * step, step=step, extents=EXT, level=lv)
        if support >= 0:
            assert r["distance"] == drop * step
            seen += 1
        else:
            assert r["distance"] >= drop * step
    G, L = _scene(np.random.default_rng(2), 40)
    A, _ = OB.grid_affine(T, 40, EXT)
    occ2, lab2 = torch.from_numpy(_posed(G, 0, 1)).to(DEV), torch.from_numpy(_posed(L, 0, 1)).to(DEV)
    m = OB.placement_map(occ2, lab2, T, 1, A[:, 0], 0, EXT, 0.45)
    iu, iv = -m["offset_lo"][0], -m["offset_lo"][1]
    s2 = EXT[0] / 39
    r = OB.slide_until_contact(occ2, lab2, T, 1, A[:, 0], 39 * s2, step=s2, extents=EXT, level=0.45)
    assert int(m["support"][iu, iv]) >= 0 and r["distance"] == pytest.approx(int(m["drop"][iu, iv]) * s2, abs=1e-12)


def test_place_object_through_edited_sweep_lands_on_nothing(nets):
    _, nf, _, _ = nets
    occ, lab = _sweep(nf)
    o, l = _np(occ, lab)
    A, b = OB.grid_affine(T, DIM, EXT)
    near = A @ np.full(3, (DIM - 1) / 2.0) + b
    found = 0
    cases = []
    for lv in (_level(occ, q) for q in (0.85, 0.95, 0.99)):          # sparser sweeps leave smaller objects with room to rest
        k, c = np.unique(l[o > np.float32(lv)], return_counts=True)
        cases += [(lv, int(x), d) for x in k[np.argsort(-c, kind="stable")] for d in _downs(T, EXT)]
    for lv, label, down in cases:
        if found == 3:
            break
        r = OB.place_object(occ, lab, T, label, down, near, stable=False, extents=EXT, level=lv)
        p = r["placement"]
        if p is None:
            assert r["candidates"] == 0 and r["reason"]
            continue
        found += 1
        assert r["tested"] == 1 and p["supported"]
        eo, el = _np(*OB.edited_sweep(nf, T, [(label, p["transformation"])], DIM, EXT, lv, NEAR, FAR, NI))
        over = (o > lv) & (l != label) & (el == label) & (eo > lv)
        assert not over.any()
        e = OB.inventory_from_grid(torch.from_numpy(eo).to(DEV), torch.from_numpy(el).to(DEV), T, EXT, lv, objects=[label])[0]
        np.testing.assert_allclose(e["centre"], p["centre"], rtol=0, atol=1e-12)
        rs = OB.place_object(occ, lab, T, label, down, near, stable=True, max_tests=8, extents=EXT, level=lv)
        if rs["placement"] is not None:
            assert rs["placement"]["stable"] and rs["tested"] <= 8
        else:
            assert rs["tested"] == min(8, rs["candidates"]) and "stable" in rs["reason"]
    assert found or len(np.unique(l[o > np.float32(_level(occ))])) == 1              # one solid label: nothing to rest on


# ---- 3. rejections -----------------------------------------------------------------------------------------------------------

def test_the_library_rejects_bad_input():
    dim = 8
    occ = torch.zeros((dim,) * 3, device=DEV)
    lab = torch.zeros((dim,) * 3, device=DEV, dtype=torch.int16)
    occ[2:4, 2:4, 2:4], lab[2:4, 2:4, 2:4] = 0.9, 1
    ctx = get_context(DEV)

    def place(d=dim, level=0.45, o=occ, la=lab, contacts=False, uv=(0, 0), **kw):
        desc = _lib.Placement(label=1, axis=0, sign=-1, lift=0)
        desc.obstacles[:] = OB.ALL_LABELS
        for k, v in kw.items():
            setattr(desc, k, v)
        info = _lib.PlacementInfo()
        maps = [torch.zeros(dim * dim, dtype=t, device=DEV) for t in (torch.int32, torch.int32, torch.int16)]
        cells = np.zeros((64, 3), dtype=np.int32)
        n, dr = C.c_int64(0), C.c_int32(0)
        with pytest.raises(RuntimeError) as e:
            if contacts:
                ctx.call("dmnerf_placement_contacts", ctx.handle, _lib.ptr(o), _lib.ptr(la, torch.int16), d, level,
                         _lib.doubles(np.eye(4), 16), _lib.doubles((4.0, 4.0, 4.0), 3), C.byref(desc), uv[0], uv[1],
                         cells.ctypes.data_as(C.POINTER(C.c_int32)), 64, C.byref(n), C.byref(dr))
            else:
                ctx.call("dmnerf_placement_map", ctx.handle, _lib.ptr(o), _lib.ptr(la, torch.int16), d, level, _lib.doubles(np.eye(4), 16),
                         _lib.doubles((4.0, 4.0, 4.0), 3), C.byref(desc), _lib.ptr(maps[0], torch.int32), _lib.ptr(maps[1], torch.int32),
                         _lib.ptr(maps[2], torch.int16), C.byref(info))
        assert info.runs == 0 and not any(int(x.abs().sum()) for x in maps) and n.value == 0
        return str(e.value)

    assert "dim" in place(d=1) and "[2, 1024]" in place(d=1025)
    assert "level" in place(level=0.0) and "level" in place(level=1.0)
    assert "outside [0, 127]" in place(label=128) and "outside [0, 127]" in place(label=-1)
    assert "axis" in place(axis=3) and "sign" in place(sign=0) and "sign" in place(sign=2)
    assert "lift" in place(lift=-1) and "lift" in place(lift=dim)
    assert "lift 5 takes the object's top" in place(lift=5)
    assert "no solid points" in place(label=2)
    bad = lab.clone()
    bad[3, 4, 5] = 128
    assert "label outside [0, 127]" in place(la=bad)
    nan = occ.clone()
    nan[1, 2, 3] = float("nan")
    assert "NaN" in place(o=nan) and "NaN" in place(o=nan, contacts=True)
    assert "offset" in place(contacts=True, uv=(5, 0))
    mask = torch.zeros((dim,) * 3, dtype=torch.bool, device=DEV)
    region = OB.region_from_mask(mask, np.eye(4), (4.0, 4.0, 4.0), applies=[3])
    assert "applies" in place(piece=region.abi(127))
    with pytest.raises(ValueError, match="no solid points"):
        OB.placement_map(occ, lab, np.eye(4), 2, (-1, 0, 0), extents=(4.0, 4.0, 4.0))
    with pytest.raises(ValueError, match="out of the grid"):
        OB.placement_map(occ, lab, np.eye(4), 1, (-1, 0, 0), lift=5, extents=(4.0, 4.0, 4.0))
    with pytest.raises(ValueError, match="applies"):
        OB.placement_map(occ, lab, np.eye(4), 1, (-1, 0, 0), extents=(4.0, 4.0, 4.0), piece=region)
    m = OB.placement_map(occ, lab, np.eye(4), 1, (-1, 0, 0), extents=(4.0, 4.0, 4.0))
    assert m["runs"] == 4 and m["points"] == 8 and (m["drop"] == 2).all() and (m["support"] == -1).all()
    with pytest.raises(ValueError, match="outside"):
        OB.placement(m, 7, 0)


# ---- 4. tools ----------------------------------------------------------------------------------------------------------------

def _checkpoint(tmp_path):
    nc, nf, _, _ = make_models(7, 8, 13, "cpu", trained_like=True)
    torch.save({"network_coarse_state_dict": nc.state_dict(), "network_fine_state_dict": nf.state_dict()}, tmp_path / "ck.tar")
    np.save(tmp_path / "T.npy", np.eye(4))
    return make_models(7, 8, 13, DEV, trained_like=True)[1]


def test_move_objects_place_at_and_find_objects_placements_write_what_the_library_returns(tmp_path):
    nf = _checkpoint(tmp_path)
    pose = np.eye(4, dtype=np.float32)
    pose[2, 3] = 6.0
    np.save(tmp_path / "pose.npy", pose)
    ext = (1.9, 7.0, 7.0)
    o, l = _np(*OB.occupancy_objects(nf, np.eye(4), OB.object_mask(13, keep=range(13)), 32, ext, device=DEV))
    lv = _level(torch.from_numpy(o), 0.5)
    label = _top_label(o, l, lv)
    near = [0.0, 0.5, 0.0]
    argv = [str(tmp_path / "ck.tar"), "--pose", str(tmp_path / "pose.npy"), "--hwk", "24", "32", "30", "0", "16", "0", "30", "12", "0",
            "0", "1", "--move-label", str(label), "--transform", str(tmp_path / "T.npy"), "--grid-dim", "32", "--level", repr(lv),
            "--out", str(tmp_path / "o"), "--N-test", "256", "--place-at"] + [repr(x) for x in near] + \
        ["--down", "0", "-1", "0", "--any-stability"]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "move_objects.py")] + argv, capture_output=True, text=True)
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import move_objects
    a = move_objects.parse(argv)
    _, lab_, _, region = move_objects.choose_piece(a, nf, np.eye(4), ext)
    occ, lab = OB.occupancy_objects(nf, np.eye(4), OB.object_mask(13, remove=[]), 32, ext, device=DEV)
    want = OB.place_object(occ, lab, np.eye(4), lab_, (0, -1, 0), near, stable=False, extents=ext, level=lv, piece=region)
    if want["placement"] is None:
        assert r.returncode != 0 and "no placement" in r.stderr
    else:
        assert r.returncode == 0, r.stderr[-3000:]
        info = json.loads(r.stdout.strip().splitlines()[-1])
        with open(tmp_path / "o" / "transform.json") as fh:
            assert json.load(fh) == {k: v for k, v in info.items() if k != "files"}
        p = want["placement"]
        assert info["place"] == {"offset": list(p["offset"]), "drop": p["drop"], "support": p["support"], "stable": p["stable"],
                                 "contacts": [list(c) for c in p["contacts"]]}
        assert info["transformations"][0]["transformation"] == p["transformation"]
    base = [sys.executable, os.path.join(ROOT, "tools", "find_objects.py"), str(tmp_path / "ck.tar"), "--transform",
            str(tmp_path / "T.npy"), "--grid-dim", "32", "--level", repr(lv), "--out", str(tmp_path / "f")]
    r = subprocess.run(base + ["--placements", str(label), "--down", "0", "-1", "0", "--lift", "0"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    info = json.loads(r.stdout.strip().splitlines()[-1])
    assert info["placements"] == "placements_%d.npz" % label and info["files"] == [info["placements"]]
    z = np.load(tmp_path / "f" / info["placements"])
    m = OB.placement_map(occ, lab, np.eye(4), label, (0, -1, 0), 0, ext, lv)
    for k in ("drop", "support", "contacts"):
        np.testing.assert_array_equal(z[k], m[k].cpu().numpy())
    assert tuple(z["offset_lo"]) == m["offset_lo"] and int(z["axis"]) == m["axis"] and int(z["runs"]) == m["runs"]
