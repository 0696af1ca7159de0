"""GPU: copying objects (DESIGN.md, "Copying objects") -- identity and absent copies bit for bit on every path; edited_grid,
move_overlap, the placement maps and support cells and arrange_objects against oracle/copy_oracle.py; "copy = move without
vacate" against the move path of edited_sweep, edited_grid and the moved render; the exact-grid agreement of edited_grid and
edited_sweep; the render's solid coarse samples against edited_sweep; both passes against the fp64 oracle; the copy as its own
piece in the inventory and alone in a component_region render; the library's rejections with no launch; and
tools/move_objects.py --copy and --arrange copies."""
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
from dmnerf_b200.autograd import mlp_forward_points, mlp_forward_rays
from dmnerf_b200.engine import get_context
from dmnerf_b200.render import render_rays
from dmnerf_b200.testing import make_models
from oracle import arrange_oracle as AO
from oracle import copy_oracle as CP
from oracle import dmnerf_oracle as O
from oracle import edit_sweep_oracle as E
from oracle import placement_oracle as PO
from oracle import render_moves_oracle as RM

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
NEAR, FAR, NI = 4.0, 15.0, 128
VOXEL = np.float32((FAR - NEAR) / NI)
T, DIM, EXT = np.eye(4), 33, (4.0, 4.0, 4.0)       # grid points and 0.125 steps are exact in fp32
MAPS = ("rgb_fine", "ins_fine", "depth_fine", "acc_fine", "weights_fine", "z_vals_fine", "rgb_coarse", "ins_coarse", "depth_coarse",
        "acc_coarse", "weights_coarse", "raw_coarse", "raw_fine")


@pytest.fixture(scope="module", params=[13, 93])
def nets(request):
    nc, nf, _, _ = make_models(101, 202, request.param, DEV)
    return nc, nf, request.param


@pytest.fixture(scope="module")
def twins(nets):
    """A coarse and a fine network with the same weights: the coarse pass then sees what edited_sweep sees."""
    _, _, ins_num = nets
    nc, nf, _, _ = make_models(303, 303, ins_num, DEV)
    return nc, nf, ins_num


def _sweep(nf, dim=DIM):
    ins_num = int(nf.ins_linear.weight.shape[0]) - 1
    with torch.no_grad():
        return OB.occupancy_objects(nf, T, OB.object_mask(ins_num, remove=[]), dim, EXT, NEAR, FAR, NI, device=DEV)


def _level(occ):
    x = occ.flatten().float()
    x = x[x > 0]
    return float(x.kthvalue(max(1, int(0.5 * x.numel()))).values)


def _top_labels(occ, labels, lv, n):
    lab = labels[occ > lv].cpu().numpy()
    k, c = np.unique(lab, return_counts=True)
    return [int(x) for x in k[np.argsort(-c, kind="stable")][:n]]


def _shift(d):
    """The move that lands an object at x + A d, d an index displacement of the dim 33 grid (0.125 per index)."""
    A, _ = OB.grid_affine(T, DIM, EXT)
    m = np.eye(4)
    m[:3, 3] = -(A @ np.asarray(d, dtype=np.float64))
    return m


def _quarter_turn(c):
    R = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    m = np.eye(4)
    m[:3, :3] = R
    m[:3, 3] = np.asarray(c) - R @ np.asarray(c)
    return m


def _np(*ts):
    return [t.cpu().numpy() for t in ts]


def _oracle_moves(o, l, lv, moves, copies, boxes=None):
    return [{"label": k, "trans": np.asarray(m, dtype=np.float64), "piece": None, "rest_drop": False, "copy": c,
             "box": E.solid_box(o, l, k, lv, 2) if boxes is None else boxes[i]}
            for i, ((k, m), c) in enumerate(zip(moves, copies))]


@pytest.fixture(scope="module")
def grid(nets):
    _, nf, _ = nets
    occ, labels = _sweep(nf)
    lv = _level(occ)
    return dict(occ=occ, labels=labels, level=lv, solid=_top_labels(occ, labels, lv, 2))


# ---- identity and absent copies -------------------------------------------------------------------------------------------------

def test_identity_and_absent_copies_change_nothing_on_the_grid_paths(nets, grid):
    _, nf, ins_num = nets
    occ, labels, lv = grid["occ"], grid["labels"], grid["level"]
    mv = grid["solid"][0]
    present = set(int(k) for k in torch.unique(labels[occ > lv]).cpu().tolist())
    absent = next(k for k in range(ins_num + 1) if k not in present)
    whole = OB.region_from_mask(torch.ones((DIM,) * 3, dtype=torch.bool, device=DEV), T, EXT, applies=[mv])
    for moves, boxes, pieces in (([(mv, np.eye(4))], None, None), ([(mv, np.eye(4))], None, [whole]),
                                 ([(absent, _shift((2, 0, 0)))], None, None), ([(mv, _shift((2, 0, 0)))], [OB.EMPTY_BOX], None)):
        o, l, _ = OB.edited_grid(occ, labels, T, moves, EXT, lv, boxes=boxes, pieces=pieces, copies=True)
        assert torch.equal(o, occ) and torch.equal(l, labels)
        with torch.no_grad():
            so, sl = OB.edited_sweep(nf, T, moves, DIM, EXT, lv, NEAR, FAR, NI, boxes=boxes, pieces=pieces, copies=True)
        assert torch.equal(so, occ) and torch.equal(sl, labels)


def _rays(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    o = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1) * 3.0
    d = (torch.rand(n, 3, generator=g) - 0.5) * 2.0 - o
    return o.to(DEV), d.to(DEV), torch.linspace(1.0, 5.0, 64).to(DEV)


@pytest.mark.parametrize("impl", [_lib.IMPL_UMMA, _lib.IMPL_UMMA_F16])
@pytest.mark.parametrize("with_piece", [False, True])
def test_identity_copy_is_the_unedited_render_bit_for_bit(nets, grid, impl, with_piece):
    nc, nf, _ = nets
    mv = grid["solid"][0]
    pieces = None
    if with_piece:
        pieces = [OB.region_from_mask(torch.ones((DIM,) * 3, dtype=torch.bool, device=DEV), T, EXT, applies=[mv])]
    moved = OB.render_moves(grid["occ"], grid["labels"], T, [(mv, np.eye(4))], EXT, grid["level"], NEAR, FAR, NI, pieces=pieces,
                            copies=True)
    assert moved.copies == (True,)
    o, d, z = _rays(512)
    with torch.no_grad():
        ref = render_rays(o, d, nc, nf, z, want_raw=True, impl=impl)
        got = render_rays(o, d, nc, nf, z, want_raw=True, impl=impl, moves=moved)
    assert got["evaluated"][0] > 0
    for k in MAPS:
        assert torch.equal(got[k], ref[k]), k


def test_absent_copies_render_nothing_new(nets, grid):
    nc, nf, ins_num = nets
    present = set(int(k) for k in torch.unique(grid["labels"][grid["occ"] > grid["level"]]).cpu().tolist())
    absent = next(k for k in range(ins_num + 1) if k not in present)
    o, d, z = _rays(256, 1)
    with torch.no_grad():
        ref = render_rays(o, d, nc, nf, z, want_raw=True)
        for moves, boxes in (([(absent, _shift((2, 0, 0)))], None), ([(grid["solid"][0], _shift((2, 0, 0)))], [OB.EMPTY_BOX])):
            moved = OB.render_moves(grid["occ"], grid["labels"], T, moves, EXT, grid["level"], NEAR, FAR, NI, boxes=boxes, copies=True)
            got = render_rays(o, d, nc, nf, z, want_raw=True, moves=moved)
            assert got["evaluated"] == (0, 0)
            for k in MAPS:
                assert torch.equal(got[k], ref[k]), k


# ---- the grid edit and the collision checks against the oracle -----------------------------------------------------------------------

def test_edited_grid_with_copies_equals_the_rule(grid):
    occ, labels, lv = grid["occ"], grid["labels"], grid["level"]
    o, l = _np(occ, labels)
    a, b = (grid["solid"] * 2)[:2]
    cases = [([(a, _shift((0, 3, 0)))], [True]),
             ([(a, _shift((0, 3, 0))), (a, _shift((0, 0, -4))), (a, _quarter_turn((0.125, -0.25, 0.0)))], [True, True, True]),
             ([(a, _shift((2, 0, 0))), (a, _shift((0, -3, 0))), (b, _shift((1, 1, 0)))], [False, True, True]),
             ([(a, _shift((0, 1, 0)))], [True])]                                                  # lands on its own source
    for moves, copies in cases:
        got_o, got_l, rep = OB.edited_grid(occ, labels, T, moves, EXT, lv, copies=copies)
        want_o, want_l, landed, over = CP.grid_edit(o, l, o, l, T, EXT, _oracle_moves(o, l, lv, moves, copies), lv)
        assert np.array_equal(got_o.cpu().numpy(), want_o) and np.array_equal(got_l.cpu().numpy(), want_l)
        assert [r["landed"] for r in rep] == landed.tolist()
        assert [r["overwritten"] for r in rep] == [{int(k): int(v[k]) for k in np.nonzero(v)[0]} for v in over]
    assert rep[0]["overwritten"].get(a, 0) > 0


def test_move_overlap_with_copies_equals_the_rule_in_the_callers_order(grid):
    occ, labels, lv = grid["occ"], grid["labels"], grid["level"]
    o, l = _np(occ, labels)
    a, b = (grid["solid"] * 2)[:2]
    moves = [(a, _shift((0, 1, 0))), (a, _shift((0, 1, 0))), (b, _shift((1, 0, 0))), (a, np.eye(4)), (b, _shift((0, 0, 2)))] * 3
    copies = [False, True, True, True, False] * 3
    got = OB.move_overlap(occ, labels, T, moves, EXT, lv, copies=copies)
    over, landed = CP.move_overlap(o, l, T, EXT, _oracle_moves(o, l, lv, moves, copies), lv)
    assert [g["landed"] for g in got] == landed.tolist()
    assert [g["overlap"] for g in got] == [{int(k): int(v[k]) for k in np.nonzero(v)[0]} for v in over]
    assert got[3]["overlap"].get(a, 0) == got[3]["landed"] > 0                 # an identity copy lies wholly on its source
    plain = OB.move_overlap(occ, labels, T, moves, EXT, lv)
    assert [p["landed"] for p in plain] == landed.tolist()
    assert all(p == g for p, g, c in zip(plain, got, copies) if not c)


def test_copy_placement_maps_and_support_cells_equal_the_rule(grid):
    occ, labels, lv = grid["occ"], grid["labels"], grid["level"]
    o, l = _np(occ, labels)
    a = grid["solid"][0]
    down = (0.0, -1.0, 0.0)
    axis, sign = PO.down_axis(T, EXT, down)
    obj = (l == a) & (o > np.float32(lv))
    top = int(np.argwhere(PO.to_columns(obj, axis, sign))[:, 2].max())
    lift = min(DIM - 1 - top, 4)
    m = OB.placement_map(occ, labels, T, a, down, lift, EXT, lv, copy=True)
    want = CP.placement_in_scene(o, l, o, l, T, EXT, a, lv, axis, sign, lift, np.eye(4), E.solid_box(o, l, a, lv, 2))
    assert m["copy"] and np.array_equal(m["drop"].cpu().numpy(), want["drop"])
    assert np.array_equal(m["support"].cpu().numpy(), want["support"])
    assert np.array_equal(m["contacts"].cpu().numpy(), want["contacts"])
    ok = np.argwhere(want["drop"] >= 0)
    for iu, iv in ok[:: max(1, len(ok) // 5)][:5]:
        u, v = int(iu) + m["offset_lo"][0], int(iv) + m["offset_lo"][1]
        p = OB.placement(m, u, v)
        cells = PO.support_cells(want, u, v)
        assert sorted(p["contacts"]) == sorted(tuple(int(x) for x in c) for c in cells)


def _table_scene(dim=17):
    """A floor (label 6), a table (label 1: a top at i 4 on four legs) and a box (label 2) on the floor."""
    occ, labels = np.zeros((dim,) * 3, dtype=np.float32), np.zeros((dim,) * 3, dtype=np.int16)
    occ[0], labels[0] = 0.9, 6
    occ[4, 6:11, 6:11], labels[4, 6:11, 6:11] = 0.9, 1
    for j in (6, 10):
        for k in (6, 10):
            occ[1:4, j, k], labels[1:4, j, k] = 0.9, 1
    occ[1:3, 1:3, 1:3], labels[1:3, 1:3, 1:3] = 0.9, 2
    return occ, labels


def test_arrangements_with_copies_equal_the_rule():
    o, l = _table_scene()
    dim = o.shape[0]
    A, b = AO.grid_affine(T, dim, EXT)
    net = lambda *i: A @ np.asarray(i, dtype=np.float64) + b                          # noqa: E731
    occ, labels = torch.from_numpy(o).to(DEV), torch.from_numpy(l).to(DEV)
    down = (-1.0, 0.0, 0.0)
    arrangements = [
        [{"label": 2, "near": net(0, 8, 3), "copy": True}, {"label": 2, "near": net(0, 8, 13), "copy": True},
         {"label": 2, "near": net(0, 3, 8), "copy": True}, {"label": 2, "near": net(0, 13, 8), "copy": True}],
        [{"label": 2, "near": net(0, 2, 2), "on": [2], "lift": 2, "copy": True}],                 # stacked on its own copy
        [{"label": 2, "near": net(0, 8, 8), "on": [1], "lift": 5}, {"label": 2, "near": net(0, 2, 14), "copy": True},
         {"label": 2, "near": net(0, 8, 8), "on": [2], "lift": 7, "copy": True}],
    ]
    for items in arrangements:
        got = OB.arrange_objects(occ, labels, T, items, down, EXT, 0.45)
        want_o, want_l, chosen = CP.arrange(o, l, T, EXT, items, down, 0.45)
        assert all(c is not None for c in chosen)
        assert np.array_equal(got["occ"].cpu().numpy(), want_o) and np.array_equal(got["labels"].cpu().numpy(), want_l)
        assert got["copies"] == [bool(it.get("copy")) for it in items]
        for it, c in zip(got["items"], chosen):
            assert it["placement"]["offset"] == c["offset"] and it["placement"]["drop"] == c["drop"]
        again, _, _ = OB.edited_grid(occ, labels, T, got["moves"], EXT, 0.45, pieces=got["pieces"], rest=got["rest"],
                                     copies=got["copies"])
        assert torch.equal(again, got["occ"])


# ---- copy = move without vacate ---------------------------------------------------------------------------------------------------

def _take_on_grid(o, l, lv, move):
    inv, b = E.grid_index_map(T, EXT, DIM)
    take, _, _ = CP.take_mask(o.reshape(-1), E.sweep_points(T, EXT, DIM), inv, b, move,
                              AO.nearest_evaluate(o, l.astype(np.int64), inv, b), lv)
    return take.reshape(o.shape)


@pytest.mark.parametrize("kind", ["translation", "quarter_turn"])
def test_a_copy_is_the_move_where_it_takes_and_the_input_elsewhere(nets, grid, kind):
    _, nf, _ = nets
    occ, labels, lv = grid["occ"], grid["labels"], grid["level"]
    o, l = _np(occ, labels)
    a = grid["solid"][0]
    trans = _shift((0, 3, -2)) if kind == "translation" else _quarter_turn((0.125, -0.25, 0.0))
    take = torch.from_numpy(_take_on_grid(o, l, lv, _oracle_moves(o, l, lv, [(a, trans)], [False])[0])).to(DEV)
    assert bool(take.any())
    with torch.no_grad():
        for copy_of, move_of in (
                (lambda: OB.edited_grid(occ, labels, T, [(a, trans)], EXT, lv, copies=True)[:2],
                 lambda: OB.edited_grid(occ, labels, T, [(a, trans)], EXT, lv)[:2]),
                (lambda: OB.edited_sweep(nf, T, [(a, trans)], DIM, EXT, lv, NEAR, FAR, NI, copies=True),
                 lambda: OB.edited_sweep(nf, T, [(a, trans)], DIM, EXT, lv, NEAR, FAR, NI))):
            co, cl = copy_of()
            mo, ml = move_of()
            assert torch.equal(co[take], mo[take]) and torch.equal(cl[take], ml[take])
            assert torch.equal(co[~take], occ[~take]) and torch.equal(cl[~take], labels[~take])
            assert not torch.equal(mo, co)                                           # the move vacated something


def _axis_rays():
    """Rays along the network x axis through every grid line's origin, depths 0 .. 4 in steps of 0.125: the coarse samples are the
    grid points of the dim 33 grid of extents 4."""
    ys = np.arange(-2.0, 2.01, 0.125)
    o = torch.tensor([[-2.0, y, zz] for y in ys for zz in ys], dtype=torch.float32, device=DEV)
    d = torch.tensor([[1.0, 0.0, 0.0]], device=DEV).expand_as(o).contiguous()
    return o, d, torch.arange(0.0, 4.0 + 1e-6, 0.125, dtype=torch.float32, device=DEV)


def _device_evaluate(model):
    def f(t, dirs):
        return mlp_forward_points(model, torch.from_numpy(t).to(DEV), torch.from_numpy(dirs).to(DEV), impl=_lib.IMPL_UMMA)
    return f


def test_the_rendered_copy_is_the_move_where_it_takes_and_the_rule(twins):
    nc, nf, _ = twins                      # one set of weights: the coarse pass sees the label the sweep found
    occ, labels = _sweep(nf)
    grid = dict(occ=occ, labels=labels, level=_level(occ))
    a = _top_labels(occ, labels, grid["level"], 1)[0]
    trans = _shift((0, 2, -1))
    o, d, z = _axis_rays()
    zz = z.expand(o.shape[0], -1)
    with torch.no_grad():
        copy = render_rays(o, d, nc, nf, z, want_raw=True,
                           moves=OB.render_moves(grid["occ"], grid["labels"], T, [(a, trans)], EXT, grid["level"], NEAR, FAR, NI,
                                                 copies=True))
        move = render_rays(o, d, nc, nf, z, want_raw=True,
                           moves=OB.render_moves(grid["occ"], grid["labels"], T, [(a, trans)], EXT, grid["level"], NEAR, FAR, NI))
        raw_c = mlp_forward_rays(nc, o, d, zz.contiguous())
        raw_f = mlp_forward_rays(nf, o, d, copy["z_vals_fine"])
    mv = [dict(label=a, trans=trans, box=E.solid_box(*_np(grid["occ"], grid["labels"]), a, grid["level"], 2), piece=None,
               rest_drop=False)]
    record = []
    RM.apply_moves(raw_c, o, d, zz, mv, T, EXT, DIM, _device_evaluate(nc), grid["level"], VOXEL, record)
    take = torch.from_numpy(record[0][0]).to(DEV).reshape(raw_c.shape[:2])
    assert bool(take.any()) and copy["evaluated"][0] == move["evaluated"][0]
    assert torch.equal(copy["raw_coarse"][take], move["raw_coarse"][take])
    assert torch.equal(copy["raw_coarse"][~take], raw_c[~take])
    copies = [dict(mv[0], copy=True)]
    want_c, _ = CP.render_apply_moves(raw_c, o, d, zz, copies, T, EXT, DIM, _device_evaluate(nc), grid["level"], VOXEL)
    want_f, _ = CP.render_apply_moves(raw_f, o, d, copy["z_vals_fine"], copies, T, EXT, DIM, _device_evaluate(nf), grid["level"], VOXEL)
    assert torch.equal(copy["raw_coarse"], want_c) and torch.equal(copy["raw_fine"], want_f)


# ---- agreement of the grid paths and the render -----------------------------------------------------------------------------------

def test_edited_grid_with_copies_equals_edited_sweep_on_the_exact_grid(nets, grid):
    _, nf, _ = nets
    occ, labels, lv = grid["occ"], grid["labels"], grid["level"]
    a, b = (grid["solid"] * 2)[:2]
    for moves, copies in (([(a, _shift((0, 3, 0)))], True),
                          ([(a, _shift((1, 0, 0))), (a, _quarter_turn((0.125, -0.25, 0.0))), (b, _shift((0, 0, 2)))],
                           [False, True, True])):
        go, gl, _ = OB.edited_grid(occ, labels, T, moves, EXT, lv, copies=copies)
        with torch.no_grad():
            so, sl = OB.edited_sweep(nf, T, moves, DIM, EXT, lv, NEAR, FAR, NI, copies=copies)
        assert torch.equal(go, so) and torch.equal(gl, sl)


def test_rendered_solid_samples_equal_the_edited_sweep_with_copies(twins):
    nc, nf, _ = twins
    occ, labels = _sweep(nf)
    lv = _level(occ)
    a = _top_labels(occ, labels, lv, 1)[0]
    moves, copies = [(a, _shift((0, 2, 0))), (a, _shift((0, 0, -3)))], [True, True]
    with torch.no_grad():
        e_occ, e_lab = OB.edited_sweep(nf, T, moves, DIM, EXT, lv, NEAR, FAR, NI, copies=copies)
        o, d, z = _axis_rays()
        got = render_rays(o, d, nc, nf, z, want_raw=True,
                          moves=OB.render_moves(occ, labels, T, moves, EXT, lv, NEAR, FAR, NI, copies=copies))
    raw = got["raw_coarse"]
    solid = (RM.occupancy(raw[..., 3], VOXEL) > lv).cpu().numpy()
    lab = torch.argmax(torch.sigmoid(raw[..., 4:]), -1).cpu().numpy()
    on = o.cpu().numpy()
    j = np.rint((on[:, 2] + 2.0) * 8).astype(int)
    k = np.rint((2.0 - on[:, 1]) * 8).astype(int)
    g_solid = (e_occ > lv).cpu().numpy()[:, j, k].T
    assert np.array_equal(solid, g_solid)
    assert np.array_equal(lab[solid], e_lab.cpu().numpy()[:, j, k].T[g_solid])
    assert not np.array_equal(g_solid, (occ > lv).cpu().numpy()[:, j, k].T)


# ---- the fp64 oracle ------------------------------------------------------------------------------------------------------------
FLOOR = 0.1                                                           # of each map's scale, as test_gpu_render_moves
AMBIGUOUS_CAP = 0.01                                                  # of the rays


@pytest.mark.parametrize("mode", ["rotation", "scale"])
def test_copies_against_the_fp64_oracle(nets, mode):
    """A manipulation_transform copy (a 90 degree yaw or a 1.2 scale about the label's centre, which lands on its source): the
    edited raw of both passes equals the copy rule on the device network bit for bit, and every map and weight is within 1e-4
    (floor: a tenth of the map's scale) of the fp64 network and composite on the kernel's own depths, a ray set aside only where
    the fp64 decisions differ from the device's (DESIGN.md section 22), at most 1 % of the rays."""
    nc, nf, ins_num = nets
    _, _, wc, wf = make_models(101, 202, ins_num, DEV)
    occ, labels = _sweep(nf, 64)
    lv = _level(occ)
    a = _top_labels(occ, labels, lv, 1)[0]
    A, b = OB.grid_affine(T, 64, EXT)
    centre = A @ torch.nonzero((labels == a) & (occ > lv)).double().mean(0).cpu().numpy() + b
    trans = np.asarray(OB.manipulation_transform(centre, mode)["transformations"][0]["transformation"])
    moved = OB.render_moves(occ, labels, T, [(a, trans)], EXT, lv, NEAR, FAR, NI, copies=True)
    om = [dict(label=a, trans=trans, box=moved.boxes[0], piece=None, rest_drop=False, copy=True)]
    o, d, z = _rays(513, 4)
    with torch.no_grad():
        got = render_rays(o, d, nc, nf, z, want_raw=True, moves=moved)
        zc, zf = got["z_vals_coarse"], got["z_vals_fine"]
        rec32 = {"coarse": [], "fine": []}
        for tag, net, zz in (("coarse", nc, zc), ("fine", nf, zf)):
            raw32 = mlp_forward_rays(net, o, d, zz)
            want, ev = CP.render_apply_moves(raw32, o, d, zz, om, T, EXT, 64, _device_evaluate(net), lv, VOXEL, rec32[tag])
            assert torch.equal(got["raw_" + tag], want), tag
            assert got["evaluated"][0 if tag == "coarse" else 1] == ev
        p64 = [{k: v.to(DEV) for k, v in O.to_torch(w, torch.float64).items()} for w in (wc, wf)]
        rec64 = {}
        ref = CP.render_on_depths(o, d, p64[0], p64[1], zc, zf, om, T, EXT, 64, lv, VOXEL, rec64)
    n = o.shape[0]
    aside = np.zeros(n, dtype=bool)
    for tag, s in (("coarse", zc.shape[1]), ("fine", zf.shape[1])):
        for (t32, v32), (t64, v64) in zip(rec32[tag], rec64[tag]):
            aside |= ((t32 != t64) | (v32 != v64)).reshape(n, s).any(-1)
    assert aside.sum() <= AMBIGUOUS_CAP * n, int(aside.sum())
    assert got["evaluated"][1] > 0 and any(t.any() for t, _ in rec32["fine"])
    keep = torch.from_numpy(~aside).to(DEV)
    for tag in ("coarse", "fine"):
        for m in ("rgb", "depth", "acc", "ins", "weights"):
            g, r = got[m + "_" + tag].double()[keep], ref[m + "_" + tag][keep]
            scale = float(r.abs().max())
            err = float(((g - r).abs() / torch.clamp(r.abs(), min=FLOOR * scale)).max())
            assert err <= 1e-4, (tag, m, err)


# ---- the copy as a piece of its own ------------------------------------------------------------------------------------------------

def test_the_inventory_reports_a_copy_apart_from_its_source_at_its_moved_centre():
    """A copy that does not touch its source is a second connected piece of the label, centred at trans^-1 . centre; a copy that
    touches its source joins it in one piece (DESIGN.md section 23)."""
    o, l = _table_scene()
    dim = o.shape[0]
    occ, labels = torch.from_numpy(o).to(DEV), torch.from_numpy(l).to(DEV)
    A, _ = OB.grid_affine(T, dim, EXT)
    src = OB.inventory_from_grid(occ, labels, T, EXT, 0.45, objects=[2])[0]
    for d, pieces in (((0, 8, 8), 2), ((3, 0, 0), 2), ((2, 0, 0), 1), ((0, 1, 0), 1)):     # (2, 0, 0) sits right on the source
        trans = np.eye(4)
        trans[:3, 3] = -(A @ np.asarray(d, dtype=np.float64))
        go, gl, _ = OB.edited_grid(occ, labels, T, [(2, trans)], EXT, 0.45, copies=True)
        inv = OB.inventory_from_grid(go, gl, T, EXT, 0.45, objects=[2], components="split")
        assert len(inv) == pieces, d
        if pieces == 1:
            continue
        want = (np.linalg.inv(trans) @ np.append(src["centre"], 1.0))[:3]
        by_distance = sorted(inv, key=lambda e: np.linalg.norm(np.asarray(e["centre"]) - src["centre"]))
        assert np.abs(np.asarray(by_distance[0]["centre"]) - src["centre"]).max() <= 1e-12
        assert np.abs(np.asarray(by_distance[1]["centre"]) - want).max() <= 1e-12
        assert by_distance[0]["voxels"] == by_distance[1]["voxels"] == src["voxels"]
        assert by_distance[0]["component"] != by_distance[1]["component"]


def test_a_component_region_of_the_edited_grid_renders_the_copy_alone(twins):
    """The largest piece of a label copied one voxel clear of every solid point of its label: in the edited sweep the copy is a
    component of its own, and a component_region of it renders the copy and drops the source.  On the axis rays every coarse
    sample is a grid point: the source's solid samples keep their label and are dropped by the region, the copy's are kept; each
    pass's maps are the composite of the region-free render's edited raw with exactly the region's samples dropped (1e-5)."""
    from oracle import objects_oracle as OO
    from oracle import region_oracle as RO
    nc, nf, ins_num = twins
    occ, labels = _sweep(nf)
    x = occ.flatten()
    x = x[x > 0]
    lv = float(x.kthvalue(int(0.98 * x.numel())).values)            # a high level: small pieces with room between them
    cc0 = OB.object_components(occ, labels, lv, 26)
    j = int(np.argmax(cc0["voxels"]))
    a = int(cc0["label"][j])
    src = cc0["grid"] == j
    solid_a = (labels == a) & (occ > lv)
    near_a = torch.nn.functional.max_pool3d(solid_a.float()[None, None], 3, 1, 1)[0, 0] > 0
    idx = torch.nonzero(src)
    shift = None
    for dist in range(3, DIM):
        for ax in range(3):
            for sgn in (1, -1):
                dd = [0, 0, 0]
                dd[ax] = sgn * dist
                q = idx + torch.tensor(dd, device=DEV)
                if shift is None and bool(((q >= 0) & (q < DIM)).all()) and not bool(near_a[q[:, 0], q[:, 1], q[:, 2]].any()):
                    shift, dst_idx = dd, q
    assert shift is not None, "no place one voxel clear of label %d for its largest piece" % a
    dst = torch.zeros_like(src)
    dst[dst_idx[:, 0], dst_idx[:, 1], dst_idx[:, 2]] = True
    piece = OB.component_region(cc0, [j], T, EXT, dilate=0)
    trans = _shift(shift)
    with torch.no_grad():
        e_occ, e_lab = OB.edited_sweep(nf, T, [(a, trans)], DIM, EXT, lv, NEAR, FAR, NI, pieces=[piece], copies=True)
    cc = OB.object_components(e_occ, e_lab, lv, 26)
    copy_ids = torch.unique(cc["grid"][dst]).cpu().tolist()
    assert len(copy_ids) == 1 and copy_ids[0] >= 0
    c = copy_ids[0]
    assert int(cc["voxels"][c]) == int(src.sum()) and torch.equal(cc["grid"] == c, dst)
    assert torch.equal(e_lab[src], labels[src]) and torch.equal(e_occ[src], occ[src])        # the source stays
    region = OB.component_region(cc, [c], T, EXT, dilate=1)
    moved = OB.render_moves(occ, labels, T, [(a, trans)], EXT, lv, NEAR, FAR, NI, pieces=[piece], copies=True)
    o, d, z = _axis_rays()
    with torch.no_grad():
        free = render_rays(o, d, nc, nf, z, want_raw=True, moves=moved)
        got = render_rays(o, d, nc, nf, z, want_raw=True, moves=moved, region=region)
    assert torch.equal(got["raw_coarse"], free["raw_coarse"])
    excl = RO.exclusion(region.voxel_map, region.bits.cpu().numpy(), DIM, region.applies_words(ins_num), True, o.cpu().numpy(),
                        d.cpu().numpy())
    for tag in ("coarse", "fine"):
        raw, zz = got["raw_" + tag], got["z_vals_" + tag]
        ex = excl(zz, OO.object_labels(raw))
        rgb, w, depth, ins, acc = O.composite(RO.exclude_samples(raw, ex), zz, d)
        for m, want in (("rgb", rgb), ("weights", w), ("depth", depth), ("ins", ins), ("acc", acc)):
            assert float((got[m + "_" + tag] - want).abs().max()) <= 1e-5 * max(1.0, float(want.abs().max())), (tag, m)
        if tag == "coarse":
            ex_c, raw_c = np.asarray(ex.cpu() if torch.is_tensor(ex) else ex), raw
    on = o.cpu().numpy()
    jr = np.rint((on[:, 2] + 2.0) * 8).astype(int)
    kr = np.rint((2.0 - on[:, 1]) * 8).astype(int)
    src_s, dst_s = src.cpu().numpy()[:, jr, kr].T, dst.cpu().numpy()[:, jr, kr].T
    lab = torch.argmax(torch.sigmoid(raw_c[..., 4:]), -1).cpu().numpy()
    solid = (RM.occupancy(raw_c[..., 3], VOXEL) > lv).cpu().numpy()
    assert src_s.any() and dst_s.any()
    assert (lab[src_s] == a).all() and solid[src_s].all() and ex_c[src_s].all()              # the source: rendered label a, dropped
    assert (lab[dst_s] == a).all() and solid[dst_s].all() and not ex_c[dst_s].any()          # the copy: label a, kept


# ---- the library's rejections ----------------------------------------------------------------------------------------------------

def test_the_library_rejects_bad_copy_flags_with_no_launch(nets):
    _, nf, _ = nets
    occ = torch.full((DIM,) * 3, 0.9, device=DEV)
    lab = torch.ones((DIM,) * 3, dtype=torch.int16, device=DEV)
    ctx = get_context(torch.device(DEV))
    shift = _shift((1, 0, 0))

    def descs(n, rest_drop=0):
        d = (_lib.EditMove * n)()
        for i in range(n):
            d[i].label, d[i].rest_drop = 1, rest_drop
            d[i].trans[:] = shift[:3].reshape(-1).tolist()
            d[i].box[:] = [0, DIM - 1] * 3
        return d

    landed, over = np.zeros(2, dtype=np.int64), np.zeros((2, 128), dtype=np.int64)
    out = (landed.ctypes.data_as(C.POINTER(C.c_int64)), over.ctypes.data_as(C.POINTER(C.c_int64)))
    state = (occ.clone(), lab.clone())
    slot = ctx.slot_for(nf)
    ctx.bind(slot, nf)
    torch.cuda.synchronize()
    before = _lib.launch_count()
    for flags, rest, msg in (([2, 0], 0, "not 0 or 1"), ([1, 0], 1, "cannot drop"), ([1, 0], 0, "follows copy")):
        with pytest.raises(RuntimeError, match=msg):
            ctx.call("dmnerf_grid_edit_copies", ctx.handle, _lib.ptr(occ), _lib.ptr(lab, torch.int16), DIM, 0.45, _lib.doubles(T, 16),
                     _lib.doubles(EXT, 3), descs(2, rest), (C.c_int32 * 2)(*flags), 2, _lib.ptr(state[0]),
                     _lib.ptr(state[1], torch.int16), *out)
        if msg != "follows copy":                   # candidates are each checked on their own: no order rule
            with pytest.raises(RuntimeError, match=msg):
                ctx.call("dmnerf_move_overlap_copies", ctx.handle, _lib.ptr(occ), _lib.ptr(lab, torch.int16), DIM, 0.45,
                         _lib.doubles(T, 16), _lib.doubles(EXT, 3), descs(2, rest), (C.c_int32 * 2)(*flags), 2, None, out[1], out[0])
        with pytest.raises(RuntimeError, match=msg):
            ctx.call("dmnerf_mesh_occupancy_edit_copies", ctx.handle, slot, _lib.doubles(T, 16), _lib.doubles(EXT, 3), DIM, float(VOXEL),
                     0.45, 0, descs(2, rest), (C.c_int32 * 2)(*flags), 2, _lib.ptr(state[0]), _lib.ptr(state[1], torch.int16),
                     C.byref(C.c_int64(0)))
    assert torch.equal(state[0], occ) and torch.equal(state[1], lab)
    p = _lib.Placement(label=1, rest_drop=1, axis=1, sign=-1, lift=0)
    p.obstacles[:] = OB.ALL_LABELS
    drop = torch.empty(DIM * DIM, dtype=torch.int32, device=DEV)
    sup = torch.empty(DIM * DIM, dtype=torch.int16, device=DEV)
    info, status = _lib.PlacementInfo(), np.zeros(1, dtype=np.int32)
    for copy, rest, msg in ((2, 0, "not 0 or 1"), (1, 1, "cannot drop")):
        p.rest_drop = rest
        with pytest.raises(RuntimeError, match=msg):
            ctx.call("dmnerf_placement_maps_in_scene_copy", ctx.handle, _lib.ptr(occ), _lib.ptr(lab, torch.int16), _lib.ptr(occ),
                     _lib.ptr(lab, torch.int16), DIM, 0.45, _lib.doubles(T, 16), _lib.doubles(EXT, 3), C.byref(p), copy,
                     _lib.doubles(np.eye(4)[:3], 12), (C.c_int32 * 6)(*([0, DIM - 1] * 3)), 1, _lib.ptr(drop, torch.int32),
                     _lib.ptr(drop, torch.int32), _lib.ptr(sup, torch.int16), C.byref(info), status.ctypes.data_as(C.POINTER(C.c_int32)))
    assert _lib.launch_count() == before
    with pytest.raises(ValueError, match="follows copy"):
        OB.edited_grid(occ, lab, T, [(1, shift)] * 2, EXT, copies=[True, False])
    with pytest.raises(ValueError, match="drop"):
        OB.move_overlap(occ, lab, T, [(1, shift)], EXT, rest="drop", copies=True)
    with pytest.raises(ValueError, match="follows copy"):
        OB.edited_sweep(nf, T, [(1, shift)] * 2, DIM, EXT, copies=[True, False])


# ---- the tool ---------------------------------------------------------------------------------------------------------------------

def test_move_objects_copies_with_the_per_sample_render(nets, tmp_path):
    nc, nf, _ = nets
    ck = tmp_path / "ck.tar"
    torch.save({"network_coarse_state_dict": {k: v.cpu() for k, v in nc.state_dict().items()},
                "network_fine_state_dict": {k: v.cpu() for k, v in nf.state_dict().items()}}, str(ck))
    np.save(str(tmp_path / "pose.npy"), np.eye(4, dtype=np.float32)[:3])
    np.save(str(tmp_path / "T.npy"), T)
    occ, lab = _sweep(nf)
    lv = _level(occ)
    ins_num = int(nf.ins_linear.weight.shape[0]) - 1
    label = next(k for k in _top_labels(occ, lab, lv, 6) if k != ins_num)
    base = [sys.executable, os.path.join(ROOT, "tools", "move_objects.py"), str(ck), "--pose", str(tmp_path / "pose.npy"), "--hwk", "8",
            "8", "10", "0", "4", "0", "10", "4", "0", "0", "1", "--transform", str(tmp_path / "T.npy"), "--extents", "4", "4", "4",
            "--grid-dim", str(DIM), "--level", str(lv), "--dilate", "0", "--N-test", "64"]
    r = subprocess.run(base + ["--move-label", str(label), "--mode", "translation", "--copy", "--check", "--out", str(tmp_path / "a")],
                       capture_output=True, text=True, cwd=ROOT)
    assert "--render samples" in r.stderr and r.returncode != 0                    # the exchanger renders moves only
    r = subprocess.run(base + ["--move-label", str(label), "--mode", "translation", "--copy", "--check", "--render", "samples",
                               "--out", str(tmp_path / "a")], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    rec = json.loads(open(tmp_path / "a" / "transform.json").read())
    assert rec["copies"] == [True] and rec["render"] == "samples" and len(rec["evaluated"]) == 2 and rec["landed"] > 0
    # --arrange: a copy of the largest piece at a high level, where small pieces leave room to set a copy down beside its source
    x = occ.flatten()
    x = x[x > 0]
    hi = float(x.kthvalue(int(0.98 * x.numel())).values)
    keep = OB.object_mask(ins_num, keep=range(ins_num))
    with torch.no_grad():
        o_obj, l_obj = OB.occupancy_objects(nf, T, keep, DIM, EXT, NEAR, FAR, NI, device=DEV)
    cc = OB.object_components(o_obj, l_obj, hi, 26)
    piece = int(np.argmax(cc["voxels"]))
    A, b = OB.grid_affine(T, DIM, EXT)
    spec = [{"piece": piece, "near": (A @ np.array([16.0, 16.0, 16.0]) + b).tolist(), "any_stability": True, "copy": True}]
    (tmp_path / "spec.json").write_text(json.dumps(spec))
    base[base.index("--level") + 1] = str(hi)
    r = subprocess.run(base + ["--arrange", str(tmp_path / "spec.json"), "--down", "0", "-1", "0", "--out", str(tmp_path / "b")],
                       capture_output=True, text=True, cwd=ROOT)
    assert "--render samples" in r.stderr and r.returncode != 0
    r = subprocess.run(base + ["--arrange", str(tmp_path / "spec.json"), "--down", "0", "-1", "0", "--render", "samples", "--out",
                               str(tmp_path / "b")], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    rec = json.loads(open(tmp_path / "b" / "transform.json").read())
    e = rec["arrange"][0]
    assert rec["copies"] == [True] and e["copy"] and e["placed"] and e["piece"] == piece
    assert len(rec["transformations"]) == 1 and len(rec["evaluated"]) == 2
    # the record's move, applied as a copy by the library, keeps the source and lands the piece where the tool placed it
    region = OB.component_region(cc, [piece], T, EXT, dilate=0)
    keep_all = OB.object_mask(ins_num, remove=[])
    with torch.no_grad():
        o_all, l_all = OB.occupancy_objects(nf, T, keep_all, DIM, EXT, NEAR, FAR, NI, device=DEV)
    trans = rec["transformations"][0]["transformation"]
    go, gl, rep = OB.edited_grid(o_all, l_all, T, [(e["label"], trans)], EXT, hi, pieces=[region], copies=True)
    src = cc["grid"] == piece
    assert torch.equal(gl[src], l_all[src]) and torch.equal(go[src], o_all[src])
    assert rep[0]["landed"] == int(cc["voxels"][piece])
    assert {int(k): v for k, v in e["overwritten"].items()} == rep[0]["overwritten"]
