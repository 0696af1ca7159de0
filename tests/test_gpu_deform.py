"""GPU: deforming objects (DESIGN.md, "Deforming objects") -- the identity table and a constant quarter turn plus translation are
the rigid move bit for bit on every path (edited sweep, edited_grid, move_overlap, the moved render's two passes); an integer
shear and twist / taper tables, alone, copied and grouped, against oracle/deform_oracle.py in edited_grid and move_overlap (whose
destination culling must match the oracle's whole-grid counts); the deformed edited sweep and moved render against the rule on
the device network and against the fp64 oracle; render samples on grid points against edited_grid; and the tool."""
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
from dmnerf_b200.render import render_rays
from dmnerf_b200.testing import make_models
from oracle import deform_oracle as DO
from oracle import dmnerf_oracle as O
from oracle import render_moves_oracle as RM
from test_gpu_collide import _checkpoint, _level, _np, _solid_labels
from test_gpu_group import (AMBIGUOUS_CAP, DEV, DIM, EXT, FAR, FLOOR_SCALE, NEAR, NI, VOXEL, T, _device_evaluate,
                            _quarter_turn, _rays, _shift, _sweep, _two_label_level, grid, nets)   # noqa: F401 (fixtures)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UP, FWD = (0.0, 0.0, 1.0), (1.0, 0.0, 0.0)                  # network z is index axis 1, network x index axis 0
IDENTITY = OB.Deformation((0.0, 0.0, 0.0), UP, FWD, -2.0, 0.5, [np.eye(2)] * 9, np.zeros((9, 2)))


def _quarter_table():
    """A constant quarter turn about the grid point c plus a translation t, and the rigid move that equals it."""
    c, t = np.array([0.125, -0.25, 0.0]), np.array([0.25, -0.125])
    Aq = np.array([[0.0, -1.0], [1.0, 0.0]])
    d = OB.Deformation(c, UP, FWD, -1.0, 0.5, [Aq] * 3, [t] * 3)
    R = np.array([[0.0, 1.0, 0.0], [-1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    m = np.eye(4)
    m[:3, :3], m[:3, 3] = R, c - R @ c - R @ np.array([t[0], t[1], 0.0])
    return d, m


def _shear_table(z0, layers, step=0.125):
    """Each layer k of height z0 + k step shifted by k grid steps along x (an integer-voxel shear)."""
    return OB.Deformation((0.0, 0.0, 0.0), UP, FWD, z0, step, [np.eye(2)] * layers,
                          np.stack([step * np.arange(layers), np.zeros(layers)], -1))


def _centre(occ, labels, label, lv, dim=DIM):
    A, b = OB.grid_affine(T, dim, EXT)
    return A @ torch.nonzero((labels == label) & (occ > lv)).double().mean(0).cpu().numpy() + b


def _all_paths(nc, nf, grid, rigid, deformed, defs, impl=_lib.IMPL_UMMA):
    """Every path of `deformed` with `defs` equals the same path of `rigid` without: sweep (and evaluated), grid edit, overlap and
    both render passes."""
    occ, labels, lv = grid["occ"], grid["labels"], grid["level"]
    boxes = OB.edit_boxes(occ, labels, rigid, T, EXT, lv)
    g = OB.edited_grid(occ, labels, T, deformed, EXT, lv, boxes=boxes, deformations=defs)
    e = OB.edited_grid(occ, labels, T, rigid, EXT, lv, boxes=boxes)
    assert torch.equal(g[0], e[0]) and torch.equal(g[1], e[1]) and g[2] == e[2]
    assert OB.move_overlap(occ, labels, T, deformed, EXT, lv, boxes=boxes, deformations=defs) == \
        OB.move_overlap(occ, labels, T, rigid, EXT, lv, boxes=boxes)
    with torch.no_grad():
        out = []
        for mv, d in ((deformed, defs), (rigid, None)):
            o, l_ = occ.clone(), labels.clone()
            n = OB.edit_occupancy(nf, T, o, l_, mv, boxes, EXT, lv, NEAR, FAR, NI, deformations=d)
            out.append((o, l_, n))
        assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1]) and out[0][2] == out[1][2]
        ro, rd, z = _rays(257, 5)
        r = [render_rays(ro, rd, nc, nf, z, want_raw=True, impl=impl,
                         moves=OB.render_moves(occ, labels, T, mv, EXT, lv, NEAR, FAR, NI, boxes=boxes, deformations=d))
             for mv, d in ((deformed, defs), (rigid, None))]
    for key in ("raw_coarse", "raw_fine", "rgb_fine", "ins_fine", "depth_fine"):
        assert torch.equal(r[0][key], r[1][key]), key
    assert r[0]["evaluated"] == r[1]["evaluated"]


@pytest.mark.parametrize("impl", [_lib.IMPL_UMMA, _lib.IMPL_UMMA_F16])
def test_the_identity_table_is_the_rigid_move_on_every_path(nets, grid, impl):
    nc, nf, _ = nets
    a = grid["pair"][0]
    moves = [(a, _shift((0, 2, -1))), (grid["pair"][1] if grid["pair"][1] is not None else a, _quarter_turn((0.125, -0.25, 0.0)))]
    _all_paths(nc, nf, grid, moves, moves, [IDENTITY, IDENTITY], impl)
    _all_paths(nc, nf, grid, moves, moves, [None, IDENTITY], impl)


def test_a_constant_quarter_turn_plus_translation_table_is_the_rigid_move_on_every_path(nets, grid):
    nc, nf, _ = nets
    a = grid["pair"][0]
    d, m = _quarter_table()
    _all_paths(nc, nf, grid, [(a, m)], [(a, np.eye(4))], [d])


# ---- the grid paths against the oracle ---------------------------------------------------------------------------------------

def _tables(occ, labels, lv, a):
    c = _centre(occ, labels, a, lv)
    return {"shear": _shear_table(-1.0, 12),
            "twist": OB.deformation(c, UP, -1.0, 1.0, 17, twist=lambda s: 75.0 * s),
            "taper": OB.deformation(c, UP, -1.0, 1.0, 9, taper=lambda s: 1.0 - 0.45 * s, bend=lambda s: 0.5 * s * s,
                                    bend_dir=(0.0, 1.0, 0.0)),
            "all": OB.deformation(c, (0.0, 0.6, 0.8), -1.2, 0.9, 33, twist=lambda s: -50.0 * s, taper=lambda s: 1.0 + 0.3 * s,
                                  bend=lambda s: 0.25 * s * s, bend_dir=(1.0, 0.0, 0.0))}


@pytest.mark.parametrize("table", ["shear", "twist", "taper", "all"])
def test_deformed_grid_edit_and_overlap_equal_the_oracle(nets, grid, table):
    occ, labels, lv = grid["occ"], grid["labels"], grid["level"]
    o, l_ = occ.cpu().numpy(), labels.cpu().numpy()
    a, b = grid["pair"]
    d = _tables(occ, labels, lv, a)[table]
    cases = [([(a, _shift((0, 1, 0)))], {}, [{}], [d]),
             ([(a, _quarter_turn((0.125, -0.25, 0.0)))], {"copies": [True]}, [{"copy": True}], [d])]
    if b is not None:                                  # a group, and a rigid move followed by a deformed copy of a group
        cases.append(([(a, _shift((1, 0, 0)))], {"groups": [[a, b]]}, [{"group": [a, b]}], [d]))
        cases.append(([(b, _shift((0, 0, 2))), (a, _shift((1, 0, 0)))], {"copies": [False, True], "groups": [None, [a, b]]},
                      [{}, {"copy": True, "group": [a, b]}], [None, d]))
    for moves, kw, extra, defs in cases:
        boxes = OB.edit_boxes(occ, labels, moves, T, EXT, lv, groups=kw.get("groups"))
        om = [dict(label=k, trans=np.asarray(m, dtype=np.float64), box=tuple(int(v) for v in bx), deform=df, **x)
              for (k, m), bx, df, x in zip(moves, boxes, defs, extra)]
        go, gl, land, over = DO.grid_edit(o, l_, o, l_, T, EXT, om, lv)
        eo, el, rep = OB.edited_grid(occ, labels, T, moves, EXT, lv, boxes=boxes, deformations=defs, **kw)
        assert np.array_equal(eo.cpu().numpy(), go) and np.array_equal(el.cpu().numpy(), gl), (table, kw)
        for i in range(len(moves)):
            assert rep[i]["landed"] == land[i]
            assert rep[i]["overwritten"] == {int(k): int(over[i][k]) for k in np.nonzero(over[i])[0]}
        if table != "shear":
            assert not torch.equal(eo, OB.edited_grid(occ, labels, T, moves, EXT, lv, boxes=boxes, **kw)[0]), table
        # each candidate on its own: the culled counts against the oracle's whole grid
        want, wl = DO.move_overlap(o, l_, T, EXT, om, lv)
        got = OB.move_overlap(occ, labels, T, moves, EXT, lv, boxes=boxes, deformations=defs, copies=kw.get("copies"),
                              groups=kw.get("groups"))
        for i in range(len(moves)):
            assert got[i]["landed"] == wl[i], (table, kw, i)
            assert got[i]["overlap"] == {int(k): int(want[i][k]) for k in np.nonzero(want[i])[0]}, (table, kw, i)


def test_the_deformed_edited_sweep_takes_the_rules_decisions(nets, grid):
    """The deformed edit pass against the oracle's rule with the device network at the oracle's own targets: the decisions
    agree except where the fp32 occupancy of a target lies within rounding of the level."""
    _, nf, _ = nets
    occ, labels, lv = grid["occ"], grid["labels"], grid["level"]
    a = grid["pair"][0]
    for table in ("shear", "all"):
        d = _tables(occ, labels, lv, a)[table]
        moves = [(a, _shift((0, 1, 1)))]
        boxes = OB.edit_boxes(occ, labels, moves, T, EXT, lv)
        with torch.no_grad():
            so, sl = occ.clone(), labels.clone()
            n = OB.edit_occupancy(nf, T, so, sl, moves, boxes, EXT, lv, NEAR, FAR, NI, deformations=[d])

            def evaluate(t):
                raw = mlp_forward_points(nf, torch.from_numpy(t).to(DEV), torch.zeros(len(t), 3, device=DEV), impl=_lib.IMPL_UMMA)
                return RM.occupancy(raw[:, 3], VOXEL).cpu().numpy(), RM.object_labels(raw).cpu().numpy()
            om = [dict(label=a, trans=np.asarray(moves[0][1], dtype=np.float64), box=tuple(int(v) for v in boxes[0]), deform=d)]
            oo, ol, on = DO.edit(occ.cpu().numpy(), labels.cpu().numpy(), T, EXT, om, evaluate, lv)
        assert n == on
        bad = (so.cpu().numpy() != oo) | (sl.cpu().numpy() != ol)
        assert bad.sum() <= 1e-3 * bad.size, int(bad.sum())
        assert not np.array_equal(oo, occ.cpu().numpy())


# ---- the moved render ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("table", ["twist", "all"])
def test_the_deformed_render_equals_the_rule_and_the_fp64_oracle(nets, table):
    nc, nf, ins_num = nets
    _, _, wc, wf = make_models(101, 202, ins_num, DEV)
    occ, labels = _sweep(nf, 64)
    lv, pair = _two_label_level(occ, labels)
    if lv is None:
        x = occ.flatten().float()
        lv = float(x[x > 0].kthvalue(max(1, int(0.5 * x[x > 0].numel()))).values)
        pair = [int(torch.mode(labels[occ > lv]).values)]
    a = pair[0]
    c = _centre(occ, labels, a, lv, 64)
    d = {"twist": OB.deformation(c, UP, -1.0, 1.0, 17, twist=lambda s: 75.0 * s),
         "all": OB.deformation(c, (0.0, 0.6, 0.8), -1.2, 0.9, 33, twist=lambda s: -50.0 * s, taper=lambda s: 1.0 + 0.3 * s,
                               bend=lambda s: 0.25 * s * s, bend_dir=(1.0, 0.0, 0.0))}[table]
    trans = np.asarray(OB.manipulation_transform(c, "rotation")["transformations"][0]["transformation"])
    moved = OB.render_moves(occ, labels, T, [(a, trans)], EXT, lv, NEAR, FAR, NI, deformations=[d])
    assert moved.deformations == (d,)
    om = [dict(label=a, trans=trans, box=moved.boxes[0], deform=d)]
    o, dr, z = _rays(513, 4)
    with torch.no_grad():
        got = render_rays(o, dr, nc, nf, z, want_raw=True, moves=moved)
        zc, zf = got["z_vals_coarse"], got["z_vals_fine"]
        rec32 = {"coarse": [], "fine": []}
        for tag, net, zz in (("coarse", nc, zc), ("fine", nf, zf)):
            raw32 = mlp_forward_rays(net, o, dr, zz)
            want, ev = DO.render_apply_moves(raw32, o, dr, zz, om, T, EXT, 64, _device_evaluate(net), lv, VOXEL, rec32[tag])
            assert torch.equal(got["raw_" + tag], want), tag
            assert got["evaluated"][0 if tag == "coarse" else 1] == ev
        assert ev > 0
        p64 = [{k: v.to(DEV) for k, v in O.to_torch(w, torch.float64).items()} for w in (wc, wf)]
        rec64 = {}
        ref = DO.render_on_depths(o, dr, p64[0], p64[1], zc, zf, om, T, EXT, 64, lv, VOXEL, rec64)
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


def test_render_samples_on_grid_points_match_the_deformed_edited_grid(nets, grid):
    """Rays along x through grid points, coarse samples every grid step: with the fine network as both networks, a coarse
    sample's solid state and label equal the deformed edited_grid at its grid point (the network at a grid point is the sweep)."""
    _, nf, _ = nets
    occ, labels, lv = grid["occ"], grid["labels"], grid["level"]
    a = grid["pair"][0]
    d = _shear_table(-1.0, 12)
    moves = [(a, _shift((0, 1, 0)))]
    boxes = OB.edit_boxes(occ, labels, moves, T, EXT, lv)
    eo, el, _ = OB.edited_grid(occ, labels, T, moves, EXT, lv, boxes=boxes, deformations=[d])
    jk = torch.cartesian_prod(torch.arange(DIM), torch.arange(DIM))
    A, b = OB.grid_affine(T, DIM, EXT)
    ro = torch.from_numpy((np.concatenate([np.zeros((len(jk), 1)), jk.numpy()], 1) @ A.T + b).astype(np.float32)).to(DEV)
    rd = torch.tensor([[0.125, 0.0, 0.0]], device=DEV).expand(len(jk), 3).contiguous()
    z = torch.arange(64, dtype=torch.float32, device=DEV)
    with torch.no_grad():
        r = render_rays(ro, rd, nf, nf, z, want_raw=True,
                        moves=OB.render_moves(occ, labels, T, moves, EXT, lv, NEAR, FAR, NI, boxes=boxes, deformations=[d]))
    raw = r["raw_coarse"][:, :DIM]                                # samples i = 0 .. DIM - 1 lie on grid points (i, j, k)
    solid = RM.occupancy(raw[..., 3].reshape(-1), VOXEL).reshape(raw.shape[:2]) > lv
    lab = RM.object_labels(raw.reshape(-1, raw.shape[-1])).reshape(raw.shape[:2])
    g_solid = (eo > lv).permute(1, 2, 0).reshape(len(jk), DIM)
    g_lab = el.permute(1, 2, 0).reshape(len(jk), DIM).long()
    assert torch.equal(solid, g_solid)
    assert torch.equal(lab[solid], g_lab[g_solid])


# ---- the tool ------------------------------------------------------------------------------------------------------------------

def test_move_objects_twist_writes_its_files(tmp_path):
    nf = _checkpoint(tmp_path)
    pose = np.eye(4, dtype=np.float32)
    pose[2, 3] = 6.0
    np.save(tmp_path / "pose.npy", pose)
    ext = (1.9, 7.0, 7.0)
    o, l_ = _np(*OB.occupancy_objects(nf, np.eye(4), OB.object_mask(13, keep=range(13)), 32, ext, device=DEV))
    lv = _level(torch.from_numpy(o))
    label = _solid_labels(o, l_, lv, 1)[0]
    argv = [str(tmp_path / "ck.tar"), "--pose", str(tmp_path / "pose.npy"), "--hwk", "24", "32", "30", "0", "16", "0", "30", "12", "0",
            "0", "1", "--move-label", str(label), "--mode", "translation", "--distance", "0.3", "--transform", str(tmp_path / "T.npy"),
            "--grid-dim", "32", "--level", repr(lv), "--out", str(tmp_path / "o"), "--render", "samples", "--mesh", "--check",
            "--min-cluster", "1", "--twist", "40", "--taper", "0.8", "--up", "0", "0", "1", "--knots", "9"]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "move_objects.py")] + argv, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    info = json.loads(r.stdout.strip().splitlines()[-1])
    assert {"rgb.png", "instance.png", "edited.ply", "color_edited.ply", "transform.json"} <= set(info["files"])
    assert info["deformation"]["twist"] == 40.0 and info["deformation"]["knots"] == 9 and "overlap" in info
    with open(tmp_path / "o" / "transform.json") as fh:
        assert json.load(fh) == {k: v for k, v in info.items() if k != "files"}
