"""GPU: moving objects together (DESIGN.md, "Moving objects together") -- a group of one is the existing move bit for bit on every
path (edited sweep, grid edit, move_overlap, placement maps and support cells, the moved render's two passes, exact and fp16; with
and without a piece or a copy); identity and absent groups change nothing; the hand-built room against oracle/group_oracle.py;
edited_grid against edited_sweep on the exact grid; the edited sweep's solid points against the same moves one label at a time;
the moved render against the rule on the device network and against the fp64 oracle; an arrangement with a group; and the
library's rejections with no launch."""
import ctypes as C

import numpy as np
import pytest
import torch

from dmnerf_b200 import _lib
from dmnerf_b200 import objects as OB
from dmnerf_b200.autograd import mlp_forward_points, mlp_forward_rays
from dmnerf_b200.engine import get_context
from dmnerf_b200.render import bind_pair, render_rays
from dmnerf_b200.testing import make_models
from oracle import dmnerf_oracle as O
from oracle import edit_sweep_oracle as E
from oracle import group_oracle as GO
from oracle import placement_oracle as PO
from test_group_host import BOOK, CUP, DOWN, FLOOR, SHELF, TABLE, WALL, _group_box, _shifted, room

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NEAR, FAR, NI = 4.0, 15.0, 128
VOXEL = np.float32((FAR - NEAR) / NI)
T, DIM, EXT = np.eye(4), 33, (4.0, 4.0, 4.0)       # grid points and 0.125 steps are exact in fp32
ROOM_DIM, ROOM_EXT, LEVEL = 17, (4.0, 4.0, 4.0), 0.45


@pytest.fixture(scope="module", params=[13, 93])
def nets(request):
    nc, nf, _, _ = make_models(101, 202, request.param, DEV)
    return nc, nf, request.param


def _sweep(nf, dim=DIM):
    ins_num = int(nf.ins_linear.weight.shape[0]) - 1
    with torch.no_grad():
        return OB.occupancy_objects(nf, T, OB.object_mask(ins_num, remove=[]), dim, EXT, NEAR, FAR, NI, device=DEV)


def _two_label_level(occ, labels):
    """A level at which the sweep's two most frequent labels both hold solid points (None when it has one solid label at every
    level tried)."""
    x = occ.flatten().float()
    x = x[x > 0]
    for q in (0.5, 0.3, 0.7, 0.15, 0.85):
        lv = float(x.kthvalue(max(1, int(q * x.numel()))).values)
        k, c = np.unique(labels[occ > lv].cpu().numpy(), return_counts=True)
        if k.size >= 2:
            return lv, [int(v) for v in k[np.argsort(-c, kind="stable")][:2]]
    return None, None


@pytest.fixture(scope="module")
def grid(nets):
    """The sweep, a level and its most frequent solid labels: two where some level gives two, else one (pair[1] is then None)."""
    _, nf, _ = nets
    occ, labels = _sweep(nf)
    lv, pair = _two_label_level(occ, labels)
    if lv is None:
        x = occ.flatten().float()
        x = x[x > 0]
        lv = float(x.kthvalue(max(1, int(0.5 * x.numel()))).values)
        pair = [int(torch.mode(labels[occ > lv]).values), None]
    return dict(occ=occ, labels=labels, level=lv, pair=pair)


def _two(grid):
    if grid["pair"][1] is None:
        pytest.skip("the synthetic sweep holds one solid label at every level tried: a group of two labels cannot take both")
    return grid["pair"]


def _shift(d, dim=DIM):
    A, _ = OB.grid_affine(T, dim, EXT)
    m = np.eye(4)
    m[:3, 3] = -(A @ np.asarray(d, dtype=np.float64))
    return m


def _quarter_turn(c):
    R = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    m = np.eye(4)
    m[:3, :3] = R
    m[:3, 3] = np.asarray(c) - R @ np.asarray(c)
    return m


def _half_piece(a, dim=DIM, ext=EXT, k=None):
    """A piece that applies to label a alone: the grid points with index k below `k` (default dim // 2)."""
    mask = torch.zeros((dim,) * 3, dtype=torch.bool, device=DEV)
    mask[:, :, :dim // 2 if k is None else k] = True
    return OB.region_from_mask(mask, T, ext, applies=[a])


def _oracle_piece(region):
    return E.Piece(region.bits.cpu().numpy(), region.dim, region.voxel_map, region.outside == "keep")


def _device_evaluate(model):
    def f(t, dirs):
        return mlp_forward_points(model, torch.from_numpy(t).to(DEV), torch.from_numpy(dirs).to(DEV), impl=_lib.IMPL_UMMA)
    return f


def _rays(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    o = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1) * 3.0
    d = (torch.rand(n, 3, generator=g) - 0.5) * 2.0 - o
    return o.to(DEV), d.to(DEV), torch.linspace(1.0, 5.0, 64).to(DEV)


# ---- a group of one is the existing move ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["move", "piece", "copy"])
def test_a_group_of_one_is_the_existing_move_on_the_grid_paths(nets, grid, kind):
    _, nf, _ = nets
    occ, labels, lv = grid["occ"], grid["labels"], grid["level"]
    a = grid["pair"][0]
    moves = [(a, _shift((0, 2, -1))), (grid["pair"][1] if grid["pair"][1] is not None else a, _quarter_turn((0.125, -0.25, 0.0)))]
    kw = {"copies": [True, True]} if kind == "copy" else {}
    if kind == "piece":
        kw["pieces"] = [_half_piece(a), None]
    one = [[k] for k, _ in moves]
    g = OB.edited_grid(occ, labels, T, moves, EXT, lv, groups=one, **kw)
    e = OB.edited_grid(occ, labels, T, moves, EXT, lv, **kw)
    assert torch.equal(g[0], e[0]) and torch.equal(g[1], e[1]) and g[2] == e[2]
    with torch.no_grad():
        gs = OB.edited_sweep(nf, T, moves, DIM, EXT, lv, NEAR, FAR, NI, groups=one, **kw)
        es = OB.edited_sweep(nf, T, moves, DIM, EXT, lv, NEAR, FAR, NI, **kw)
    assert torch.equal(gs[0], es[0]) and torch.equal(gs[1], es[1])
    assert OB.move_overlap(occ, labels, T, moves, EXT, lv, groups=one, **kw) == OB.move_overlap(occ, labels, T, moves, EXT, lv, **kw)
    piece = kw.get("pieces", [None])[0]
    copy = kind == "copy"
    got = OB.placement_map(occ, labels, T, a, DOWN, extents=EXT, level=lv, piece=piece, copy=copy, group=[a])
    want = OB.placement_map(occ, labels, T, a, DOWN, extents=EXT, level=lv, piece=piece, copy=copy, scene=(occ, labels))
    for key in ("drop", "support", "contacts"):
        assert torch.equal(got[key], want[key]), key
    assert got["centre"] == want["centre"] and got["points"] == want["points"]
    rest = torch.nonzero((want["drop"] >= 0) & (want["support"] >= 0))
    if rest.shape[0]:
        u, v = int(rest[0, 0]) + want["offset_lo"][0], int(rest[0, 1]) + want["offset_lo"][1]
        pg, pw = OB.placement(got, u, v), OB.placement(want, u, v)
        assert pg["contacts"] == pw["contacts"] and pg["stable"] == pw["stable"]


@pytest.mark.parametrize("impl", [_lib.IMPL_UMMA, _lib.IMPL_UMMA_F16])
@pytest.mark.parametrize("kind", ["move", "piece", "copy"])
def test_a_group_of_one_is_the_existing_moved_render_bit_for_bit(nets, grid, impl, kind):
    nc, nf, _ = nets
    a = grid["pair"][0]
    moves = [(a, _shift((0, 2, -1)))]
    kw = {"copies": True} if kind == "copy" else {"pieces": [_half_piece(a)]} if kind == "piece" else {}
    o, d, z = _rays(257, 1)
    out = []
    for groups in ([[a]], None):
        m = OB.render_moves(grid["occ"], grid["labels"], T, moves, EXT, grid["level"], NEAR, FAR, NI, groups=groups, **kw)
        with torch.no_grad():
            out.append(render_rays(o, d, nc, nf, z, want_raw=True, impl=impl, moves=m))
    for key in ("raw_coarse", "raw_fine", "rgb_fine", "ins_fine", "depth_fine"):
        assert torch.equal(out[0][key], out[1][key]), key
    assert out[0]["evaluated"] == out[1]["evaluated"]


def test_identity_and_absent_groups_change_nothing(nets, grid):
    nc, nf, ins_num = nets
    occ, labels, lv = grid["occ"], grid["labels"], grid["level"]
    present = set(int(k) for k in torch.unique(labels[occ > lv]).cpu().tolist())
    absent = [k for k in range(ins_num + 1) if k not in present][:2]
    whole = [k for k in grid["pair"] if k is not None]
    for moves, groups in (([(whole[0], np.eye(4))], [whole + absent[:1]]), ([(absent[0], _shift((2, 0, 0)))], [absent])):
        o, l, _ = OB.edited_grid(occ, labels, T, moves, EXT, lv, groups=groups)
        assert torch.equal(o, occ) and torch.equal(l, labels)
        with torch.no_grad():
            so, sl = OB.edited_sweep(nf, T, moves, DIM, EXT, lv, NEAR, FAR, NI, groups=groups)
        assert torch.equal(so, occ) and torch.equal(sl, labels)
        o, d, z = _rays(129, 2)
        with torch.no_grad():
            got = render_rays(o, d, nc, nf, z, want_raw=True,
                              moves=OB.render_moves(occ, labels, T, moves, EXT, lv, NEAR, FAR, NI, groups=groups))
            plain = render_rays(o, d, nc, nf, z, want_raw=True)
        assert torch.equal(got["rgb_fine"], plain["rgb_fine"]) and torch.equal(got["raw_coarse"], plain["raw_coarse"])


# ---- the hand-built room against the oracle ---------------------------------------------------------------------------------------

def _room_on_device():
    occ, labels = room()
    return occ, labels, torch.from_numpy(occ).to(DEV), torch.from_numpy(labels).to(DEV)


def _room_shift(d):
    A, _ = OB.grid_affine(T, ROOM_DIM, ROOM_EXT)
    m = np.eye(4)
    m[:3, 3] = -(A @ np.asarray(d, dtype=np.float64))
    return m


def test_the_room_on_the_grid_paths_equals_the_oracle():
    o, l, occ, labels = _room_on_device()
    c = OB.carried_labels(occ, labels, T, TABLE, DOWN, ROOM_EXT, LEVEL, exclude=[WALL])
    assert c["group"] == [TABLE, CUP, BOOK] and c["chain"][BOOK][0] == CUP
    assert WALL in OB.carried_labels(occ, labels, T, TABLE, DOWN, ROOM_EXT, LEVEL)["group"]
    group = c["group"]
    for d, copy in (((0, 0, 6), False), ((0, 0, 8), True), ((1, 0, 0), False)):
        trans = _room_shift(d)
        om = [{"label": TABLE, "group": group, "trans": trans, "box": _group_box(o, l, group), "copy": copy}]
        go, gl, land, over = GO.grid_edit(o, l, o, l, T, ROOM_EXT, om, LEVEL)
        eo, el, rep = OB.edited_grid(occ, labels, T, [(TABLE, trans)], ROOM_EXT, LEVEL, copies=copy, groups=[group])
        assert np.array_equal(eo.cpu().numpy(), go) and np.array_equal(el.cpu().numpy(), gl)
        assert rep[0]["landed"] == land[0] and rep[0]["overwritten"] == {int(k): int(over[0][k]) for k in np.nonzero(over[0])[0]}
        want, wl = GO.move_overlap(o, l, T, ROOM_EXT, om, LEVEL)
        got = OB.move_overlap(occ, labels, T, [(TABLE, trans)], ROOM_EXT, LEVEL, copies=copy, groups=[group])[0]
        assert got["landed"] == wl[0] and got["overlap"] == {int(k): int(want[0][k]) for k in np.nonzero(want[0])[0]}
    shelf = OB.move_overlap(occ, labels, T, [(TABLE, _room_shift((0, 0, 6)))], ROOM_EXT, LEVEL, groups=[group])[0]
    assert shelf["overlap"] == {SHELF: 4}
    before = OB.inventory_from_grid(occ, labels, T, ROOM_EXT, LEVEL, objects=group)
    eo, el, _ = OB.edited_grid(occ, labels, T, [(TABLE, _room_shift((0, 0, 6)))], ROOM_EXT, LEVEL, groups=[group])
    after = OB.inventory_from_grid(eo, el, T, ROOM_EXT, LEVEL, objects=group)
    A, _ = OB.grid_affine(T, ROOM_DIM, ROOM_EXT)
    for x, y in zip(before, after):
        np.testing.assert_allclose(np.asarray(y["centre"]) - np.asarray(x["centre"]), A @ np.array([0.0, 0.0, 6.0]), rtol=0,
                                   atol=1e-12)


def test_the_room_with_a_piece_of_the_table_equals_the_oracle_on_the_grid_paths():
    """A piece that applies to the table alone (the grid points k <= 5, which split the cup and the book at k 5 | 6) cuts the
    table and leaves the cup and the book whole: the piece is tested with the label of each point, in edited_grid, move_overlap
    and placement, each with its default box (the table's piece, the cup and the book, grown by 2).  A piece tested with the
    move's label instead would cut the cup and the book too."""
    o, l, occ, labels = _room_on_device()
    group = [TABLE, CUP, BOOK]
    region = _half_piece(TABLE, ROOM_DIM, ROOM_EXT, k=6)
    half = np.zeros((ROOM_DIM,) * 3, dtype=bool)
    half[:, :, :6] = True
    cut = (np.isin(l, [CUP, BOOK]) | ((l == TABLE) & half)) & (o > np.float32(LEVEL))
    idx = np.argwhere(cut)
    box = tuple(int(x) for a in range(3) for x in (max(idx[:, a].min() - 2, 0), min(idx[:, a].max() + 2, ROOM_DIM - 1)))
    got_box = OB.edit_boxes(occ, labels, [(TABLE, np.eye(4))], T, ROOM_EXT, LEVEL, pieces=[region], groups=[group])
    assert tuple(int(x) for x in got_box[0]) == box
    piece = _oracle_piece(region)
    for d, rest, copy in (((0, 0, 8), "keep", False), ((0, 0, 8), "drop", False), ((1, 0, 6), "keep", True)):
        trans = _room_shift(d)
        om = [{"label": TABLE, "group": group, "trans": trans, "box": box, "piece": piece, "applies": [TABLE],
               "rest_drop": rest == "drop", "copy": copy}]
        go, gl, land, over = GO.grid_edit(o, l, o, l, T, ROOM_EXT, om, LEVEL)
        eo, el, rep = OB.edited_grid(occ, labels, T, [(TABLE, trans)], ROOM_EXT, LEVEL, pieces=[region], rest=rest, copies=copy,
                                     groups=[group])
        assert np.array_equal(eo.cpu().numpy(), go) and np.array_equal(el.cpu().numpy(), gl), (d, rest, copy)
        assert rep[0]["landed"] == land[0] and rep[0]["overwritten"] == {int(k): int(over[0][k]) for k in np.nonzero(over[0])[0]}
        for k in (CUP, BOOK):                          # the piece does not apply to them: they land whole
            src = (l == k) & (o > np.float32(LEVEL))
            want = _shifted(src, d) | (src if copy else False)
            assert np.array_equal((el.cpu().numpy() == k) & (eo.cpu().numpy() > np.float32(LEVEL)), want), (k, d, rest, copy)
        want, wl = GO.move_overlap(o, l, T, ROOM_EXT, om, LEVEL)
        got = OB.move_overlap(occ, labels, T, [(TABLE, trans)], ROOM_EXT, LEVEL, pieces=[region], rest=rest, copies=copy,
                              groups=[group])[0]
        assert got["landed"] == wl[0] and got["overlap"] == {int(k): int(want[0][k]) for k in np.nonzero(want[0])[0]}
    axis, sign = PO.down_axis(T, ROOM_EXT, DOWN)
    m = OB.placement_map(occ, labels, T, TABLE, DOWN, extents=ROOM_EXT, level=LEVEL, piece=region, group=group)
    assert m["box"] == box and m["points_before"] == int(cut.sum()) == m["points"]
    om = {"label": TABLE, "group": group, "trans": np.eye(4), "box": box, "piece": piece, "applies": [TABLE]}
    want = GO.placement_in_scene(o, l, o, l, T, ROOM_EXT, om, LEVEL, axis, sign, 0)
    for key in ("drop", "support", "contacts"):
        assert np.array_equal(m[key].cpu().numpy(), want[key]), key
    assert m["points"] == want["points"].shape[0]


def test_the_room_placement_of_the_group_equals_the_oracle_and_rests_on_the_floor():
    o, l, occ, labels = _room_on_device()
    group = [TABLE, CUP, BOOK]
    axis, sign = PO.down_axis(T, ROOM_EXT, DOWN)
    m = OB.placement_map(occ, labels, T, TABLE, DOWN, extents=ROOM_EXT, level=LEVEL, group=group)
    om = {"label": TABLE, "group": group, "trans": np.eye(4), "box": m["box"]}
    want = GO.placement_in_scene(o, l, o, l, T, ROOM_EXT, om, LEVEL, axis, sign, 0)
    for key in ("drop", "support", "contacts"):
        assert np.array_equal(m[key].cpu().numpy(), want[key]), key
    assert m["points"] == want["points"].shape[0]
    p = OB.placement(m, 0, 0)
    assert p["support"] == FLOOR and p["drop"] == 0 and p["stable"]
    assert not any(c[2] in group for c in p["contacts"])
    A, b = OB.grid_affine(T, ROOM_DIM, ROOM_EXT)
    r = OB.place_object(occ, labels, T, TABLE, DOWN, A @ np.array([0.0, 3.0, 3.0]) + b, on=[FLOOR], extents=ROOM_EXT, level=LEVEL,
                        group=group)
    assert r["placement"] is not None and r["placement"]["support"] == FLOOR
    with pytest.raises(ValueError, match="never rests on itself"):
        OB.place_object(occ, labels, T, TABLE, DOWN, (0, 0, 0), on=[CUP], extents=ROOM_EXT, level=LEVEL, group=group)


def test_an_arrangement_with_a_group_equals_the_grid_edit_and_renders_by_the_rule(nets):
    nc, nf, _ = nets
    o, l, occ, labels = _room_on_device()
    A, b = OB.grid_affine(T, ROOM_DIM, ROOM_EXT)
    items = [{"label": TABLE, "group": [TABLE, CUP, BOOK], "near": A @ np.array([0.0, 11.0, 11.0]) + b, "on": [FLOOR]}]
    r = OB.arrange_objects(occ, labels, T, items, DOWN, ROOM_EXT, LEVEL)
    assert r["items"][0]["placement"] is not None and r["groups"] == [(TABLE, CUP, BOOK)]
    eo, el, _ = OB.edited_grid(occ, labels, T, r["moves"], ROOM_EXT, LEVEL, pieces=r["pieces"], rest=r["rest"], copies=r["copies"],
                               groups=r["groups"])
    assert torch.equal(eo, r["occ"]) and torch.equal(el, r["labels"])
    for k in (TABLE, CUP, BOOK):
        assert int(((r["labels"] == k) & (r["occ"] > LEVEL)).sum()) == int(((labels == k) & (occ > LEVEL)).sum())
    moved = OB.render_moves(occ, labels, T, r["moves"], ROOM_EXT, LEVEL, NEAR, FAR, NI, pieces=r["pieces"], rest=r["rest"],
                            copies=r["copies"], groups=r["groups"])
    assert moved.groups == ((TABLE, CUP, BOOK),)
    o_, d_, z_ = _rays(65, 3)
    with torch.no_grad():
        got = render_rays(o_, d_, nc, nf, z_, want_raw=True, moves=moved)
        raw_c = mlp_forward_rays(nc, o_, d_, z_.expand(o_.shape[0], -1).contiguous())
    om = [{"label": TABLE, "group": [TABLE, CUP, BOOK], "trans": np.asarray(r["moves"][0][1], dtype=np.float64),
           "box": moved.boxes[0]}]
    want, _ = GO.render_apply_moves(raw_c, o_, d_, z_.expand(o_.shape[0], -1), om, T, ROOM_EXT, ROOM_DIM, _device_evaluate(nc),
                                    LEVEL, VOXEL)
    assert torch.equal(got["raw_coarse"], want)
    with torch.no_grad():
        m = OB.edited_mesh(nf, T, r["moves"], ROOM_DIM, ROOM_EXT, LEVEL, NEAR, FAR, NI, pieces=r["pieces"], rest=r["rest"],
                           copies=r["copies"], groups=r["groups"], min_cluster=1)
    assert m["labels"].shape[0] == m["clean_vertices"].shape[0]


# ---- the grid paths agree, and the group against the sequence ---------------------------------------------------------------------

def test_edited_grid_with_groups_equals_edited_sweep_on_the_exact_grid(nets, grid):
    _, nf, _ = nets
    occ, labels, lv = grid["occ"], grid["labels"], grid["level"]
    a, b = _two(grid)
    for moves, groups, copies, pieces in (([(a, _shift((0, 3, 0)))], [[a, b]], None, None),
                                          ([(a, _quarter_turn((0.125, -0.25, 0.0)))], [[a, b]], None, None),
                                          ([(a, _shift((1, 0, 0))), (b, _shift((0, 0, 2)))], [[a, b], None], [False, True], None),
                                          ([(a, _shift((0, 3, 0)))], [[a, b]], None, [_half_piece(a)])):   # the piece cuts a only
        go, gl, _ = OB.edited_grid(occ, labels, T, moves, EXT, lv, copies=copies, groups=groups, pieces=pieces)
        with torch.no_grad():
            so, sl = OB.edited_sweep(nf, T, moves, DIM, EXT, lv, NEAR, FAR, NI, copies=copies, groups=groups, pieces=pieces)
        assert torch.equal(go, so) and torch.equal(gl, sl)
        if pieces is not None:                         # the piece does not apply to b: every solid point of b lands 3 voxels along j
            want = torch.zeros_like(labels, dtype=torch.bool)
            want[:, 3:] = ((labels == b) & (occ > lv))[:, :-3]
            assert torch.equal((gl == b) & (go > lv), want)


def test_the_edited_sweep_of_a_group_has_the_solid_points_of_its_moves_in_sequence(nets, grid):
    _, nf, _ = nets
    a, b = _two(grid)
    lv = grid["level"]
    trans = _shift((0, 2, -1))
    box = tuple(OB.edit_boxes(grid["occ"], grid["labels"], [(a, trans)], T, EXT, lv, groups=[[a, b]])[0])
    with torch.no_grad():
        go, gl = OB.edited_sweep(nf, T, [(a, trans)], DIM, EXT, lv, NEAR, FAR, NI, boxes=[box], groups=[[a, b]])
        so, sl = OB.edited_sweep(nf, T, [(a, trans), (b, trans)], DIM, EXT, lv, NEAR, FAR, NI, boxes=[box, box])
    solid = go > lv
    assert torch.equal(solid, so > lv)
    assert torch.equal(go[solid], so[solid]) and torch.equal(gl[solid], sl[solid])
    assert bool(((gl == a) & solid).any()) and bool(((gl == b) & solid).any())
    assert not torch.equal(solid, grid["occ"] > lv)


# ---- the moved render: the rule on the device network, and the fp64 oracle --------------------------------------------------------
FLOOR_SCALE = 0.1                                                     # of each map's scale, as test_gpu_render_moves
AMBIGUOUS_CAP = 0.01                                                  # of the rays


@pytest.mark.parametrize("mode", ["translation", "rotation", "piece"])
def test_the_moved_render_of_a_group_equals_the_rule_and_the_fp64_oracle(nets, mode):
    nc, nf, ins_num = nets
    _, _, wc, wf = make_models(101, 202, ins_num, DEV)
    occ, labels = _sweep(nf, 64)
    lv, pair = _two_label_level(occ, labels)
    if lv is None:
        pytest.skip("the synthetic sweep holds one solid label at every level tried: a group of two labels cannot take both")
    a, b = pair
    A, bb = OB.grid_affine(T, 64, EXT)
    centre = A @ torch.nonzero(((labels == a) | (labels == b)) & (occ > lv)).double().mean(0).cpu().numpy() + bb
    kind = "translation" if mode == "piece" else mode
    trans = np.asarray(OB.manipulation_transform(centre, kind)["transformations"][0]["transformation"])
    region = _half_piece(a, 64) if mode == "piece" else None       # a piece that cuts a and leaves b whole
    moved = OB.render_moves(occ, labels, T, [(a, trans)], EXT, lv, NEAR, FAR, NI, groups=[[a, b]],
                            pieces=None if region is None else [region])
    om = [dict(label=a, group=[a, b], trans=trans, box=moved.boxes[0], piece=None if region is None else _oracle_piece(region),
               applies=[a], rest_drop=False)]
    o, d, z = _rays(513, 4)
    with torch.no_grad():
        got = render_rays(o, d, nc, nf, z, want_raw=True, moves=moved)
        zc, zf = got["z_vals_coarse"], got["z_vals_fine"]
        rec32 = {"coarse": [], "fine": []}
        for tag, net, zz in (("coarse", nc, zc), ("fine", nf, zf)):
            raw32 = mlp_forward_rays(net, o, d, zz)
            want, ev = GO.render_apply_moves(raw32, o, d, zz, om, T, EXT, 64, _device_evaluate(net), lv, VOXEL, rec32[tag])
            assert torch.equal(got["raw_" + tag], want), tag
            assert got["evaluated"][0 if tag == "coarse" else 1] == ev
        p64 = [{k: v.to(DEV) for k, v in O.to_torch(w, torch.float64).items()} for w in (wc, wf)]
        rec64 = {}
        ref = GO.render_on_depths(o, d, p64[0], p64[1], zc, zf, om, T, EXT, 64, lv, VOXEL, rec64)
    n = o.shape[0]
    aside = np.zeros(n, dtype=bool)
    for tag, s in (("coarse", zc.shape[1]), ("fine", zf.shape[1])):
        for (t32, v32), (t64, v64) in zip(rec32[tag], rec64[tag]):
            aside |= ((t32 != t64) | (v32 != v64)).reshape(n, s).any(-1)
    assert aside.sum() <= AMBIGUOUS_CAP * n, int(aside.sum())
    keep = torch.from_numpy(~aside).to(DEV)
    for tag in ("coarse", "fine"):
        for m in ("rgb", "depth", "acc", "ins", "weights"):
            g, r = got[m + "_" + tag].double()[keep], ref[m + "_" + tag][keep]
            scale = float(r.abs().max())
            err = float(((g - r).abs() / torch.clamp(r.abs(), min=FLOOR_SCALE * scale)).max())
            assert err <= 1e-4, (tag, m, err)


# ---- rejections ------------------------------------------------------------------------------------------------------------------

def test_the_library_rejects_bad_groups_with_no_launch(nets):
    nc, nf, ins_num = nets
    occ = torch.full((DIM,) * 3, 0.9, device=DEV)
    lab = torch.ones((DIM,) * 3, dtype=torch.int16, device=DEV)
    ctx = get_context(torch.device(DEV))
    shift = _shift((1, 0, 0))

    def descs(*labels):
        d = (_lib.EditMove * len(labels))()
        for i, k in enumerate(labels):
            d[i].label = k
            d[i].trans[:] = shift[:3].reshape(-1).tolist()
            d[i].box[:] = [0, DIM - 1] * 3
        return d
    d = descs(1, 1)
    landed, over = np.zeros(2, dtype=np.int64), np.zeros((2, 128), dtype=np.int64)
    out = (landed.ctypes.data_as(C.POINTER(C.c_int64)), over.ctypes.data_as(C.POINTER(C.c_int64)))
    state = (occ.clone(), lab.clone())
    bind_pair(ctx, nc, nf)
    slot = ctx.slot_for(nf)
    ctx.bind(slot, nf)
    torch.cuda.synchronize()
    before = _lib.launch_count()

    def words(*sets):
        return (C.c_uint32 * 8)(*[w for s in sets for w in OB.label_words(s)])
    out_of_net = ins_num + 1                               # beyond the network, inside the grid-only range
    # the order rule compares label sets: a move of label 2 (set {2}) after a copy of label 1 whose set holds 2
    for d, groups, flags, msg, grid_only in ((descs(1, 1), words([2], [1]), None, "does not hold the moved label 1", True),
                                             (descs(1, 1), words([1, out_of_net], [1]), None, "outside \\[0, %d\\]" % ins_num,
                                              False),
                                             (descs(1, 2), words([1, 2], [2]), (C.c_int32 * 2)(1, 0),
                                              "move 1 of label 2 follows copy 0", True)):
        if grid_only:
            with pytest.raises(RuntimeError, match="grid_edit_groups: .*" + msg):
                ctx.call("dmnerf_grid_edit_groups", ctx.handle, _lib.ptr(occ), _lib.ptr(lab, torch.int16), DIM, 0.45,
                         _lib.doubles(T, 16), _lib.doubles(EXT, 3), d, flags, groups, 2, _lib.ptr(state[0]),
                         _lib.ptr(state[1], torch.int16), *out)
        with pytest.raises(RuntimeError, match="mesh_occupancy_edit_groups: .*" + msg):
            ctx.call("dmnerf_mesh_occupancy_edit_groups", ctx.handle, slot, _lib.doubles(T, 16), _lib.doubles(EXT, 3), DIM,
                     float(VOXEL), 0.45, 0, d, flags, groups, 2, _lib.ptr(state[0]), _lib.ptr(state[1], torch.int16),
                     C.byref(C.c_int64(0)))
    d = descs(1, 1)
    with pytest.raises(RuntimeError, match="move_overlap_groups: .*does not hold"):
        ctx.call("dmnerf_move_overlap_groups", ctx.handle, _lib.ptr(occ), _lib.ptr(lab, torch.int16), DIM, 0.45, _lib.doubles(T, 16),
                 _lib.doubles(EXT, 3), d, None, words([2], [1]), 2, None, out[1], out[0])
    rm = _lib.RenderMoves()
    rm.moves, rm.n_moves, rm.dim = C.cast(d, C.POINTER(_lib.EditMove)), 2, DIM
    rm.transform[:] = T.reshape(-1).tolist()
    rm.extents[:] = list(EXT)
    rm.level, rm.voxel = 0.45, float(VOXEL)
    evaluated = (C.c_int64 * 2)()
    for groups, flags, msg in ((words([2], [1]), None, "does not hold the moved label 1"),
                               (words([1, out_of_net], [1]), None, "outside \\[0, %d\\]" % ins_num)):
        with pytest.raises(RuntimeError, match="render_moved_groups: .*" + msg):
            ctx.call("dmnerf_render_moved_groups", ctx.handle, C.byref(_lib.RenderIO()), 1, 64, 128, 0, _lib.IMPL_UMMA, C.byref(rm),
                     flags, groups, evaluated)
    with pytest.raises(RuntimeError, match="render_moved_groups: .*move 1 of label 2 follows copy 0"):
        d2 = descs(1, 2)
        rm.moves = C.cast(d2, C.POINTER(_lib.EditMove))
        ctx.call("dmnerf_render_moved_groups", ctx.handle, C.byref(_lib.RenderIO()), 1, 64, 128, 0, _lib.IMPL_UMMA, C.byref(rm),
                 (C.c_int32 * 2)(1, 0), words([1, 2], [2]), evaluated)
    p = _lib.Placement(label=1, rest_drop=0, axis=1, sign=-1, lift=0)
    p.obstacles[:] = OB.ALL_LABELS
    drop = torch.empty(DIM * DIM, dtype=torch.int32, device=DEV)
    sup = torch.empty(DIM * DIM, dtype=torch.int16, device=DEV)
    info, status = _lib.PlacementInfo(), np.zeros(1, dtype=np.int32)
    with pytest.raises(RuntimeError, match="placement_maps_in_scene_group: .*does not hold"):
        ctx.call("dmnerf_placement_maps_in_scene_group", ctx.handle, _lib.ptr(occ), _lib.ptr(lab, torch.int16), _lib.ptr(occ),
                 _lib.ptr(lab, torch.int16), DIM, 0.45, _lib.doubles(T, 16), _lib.doubles(EXT, 3), C.byref(p), 0,
                 (C.c_uint32 * 4)(*OB.label_words([2])), _lib.doubles(np.eye(4)[:3], 12), (C.c_int32 * 6)(*([0, DIM - 1] * 3)), 1,
                 _lib.ptr(drop, torch.int32), _lib.ptr(drop, torch.int32), _lib.ptr(sup, torch.int16), C.byref(info),
                 status.ctypes.data_as(C.POINTER(C.c_int32)))
    cells, got, dr = np.zeros((4, 3), dtype=np.int32), C.c_int64(0), C.c_int32(0)
    for group, msg in ((OB.label_words([2]), "does not hold the moved label 1"), ([0, 0, 0, 0], "does not hold")):
        with pytest.raises(RuntimeError, match="placement_contacts_in_scene_group: .*" + msg):
            ctx.call("dmnerf_placement_contacts_in_scene_group", ctx.handle, _lib.ptr(occ), _lib.ptr(lab, torch.int16), _lib.ptr(occ),
                     _lib.ptr(lab, torch.int16), DIM, 0.45, _lib.doubles(T, 16), _lib.doubles(EXT, 3), C.byref(p), 0,
                     (C.c_uint32 * 4)(*group), _lib.doubles(np.eye(4)[:3], 12), (C.c_int32 * 6)(*([0, DIM - 1] * 3)), 0, 0,
                     cells.ctypes.data_as(C.POINTER(C.c_int32)), 4, C.byref(got), C.byref(dr))
    assert _lib.launch_count() == before
    assert torch.equal(state[0], occ) and torch.equal(state[1], lab)
    with pytest.raises(ValueError, match="does not hold"):
        OB.move_overlap(occ, lab, T, [(1, shift)], EXT, groups=[[2]])
    with pytest.raises(ValueError, match="follows copy"):
        OB.edited_sweep(nf, T, [(1, shift), (2, shift)], DIM, EXT, copies=[True, False], groups=[[1, 2], None])
