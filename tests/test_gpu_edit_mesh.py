"""GPU: meshing an edited scene -- the edit pass (dmnerf_mesh_occupancy_edit) against the numpy rule and the fp64 network, the
vertex labels, edited_mesh and tools/move_objects.py --mesh."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from dmnerf_b200 import _lib
from dmnerf_b200 import mesh as M
from dmnerf_b200 import objects as OB
from dmnerf_b200.engine import get_context
from dmnerf_b200.testing import make_models
from oracle import dmnerf_oracle as O
from oracle import edit_sweep_oracle as E

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
QUANTILE = 0.5                       # the synthetic networks need not cross 0.45: each test's level is a quantile of its sweep
NEAR, FAR, NI = 4.0, 15.0, 128
VOXEL = (FAR - NEAR) / NI
EXACT = dict(T=np.eye(4), dim=33, ext=(4.0, 4.0, 4.0))      # grid points and 0.125 steps are exact in fp32


@pytest.fixture(scope="module", params=[13, 93])
def nets(request):
    return make_models(101, 202, request.param, DEV)


def _sweep(nf, T, dim, ext):
    ins_num = int(nf.ins_linear.weight.shape[0]) - 1
    return OB.occupancy_objects(nf, T, OB.object_mask(ins_num, remove=[]), dim, ext, NEAR, FAR, NI, device=DEV)


def _level(occ):
    """The QUANTILE of a sweep's positive occupancies (most grid points are empty), an fp32 value in (0, 1)."""
    x = occ.flatten().float()
    x = x[x > 0]
    lv = float(x.kthvalue(max(1, int(QUANTILE * x.numel()))).values)
    assert 0.0 < lv < 1.0
    return lv


def _np(*ts):
    return [t.cpu().numpy() for t in ts]


def _solid_labels(occ, labels, lv, n=3):
    """The n labels with the most solid points."""
    lab = labels[occ > np.float32(lv)]
    k, c = np.unique(lab, return_counts=True)
    return [int(x) for x in k[np.argsort(-c, kind="stable")][:n]]


def _move(label, trans, box, piece=None, rest_drop=False):
    return dict(label=label, trans=np.asarray(trans, dtype=np.float64), box=tuple(int(v) for v in box), piece=piece,
                rest_drop=rest_drop)


def _turn_about(c, k=1):
    """k quarter turns about the network z axis through c, as a 4x4."""
    R = np.linalg.matrix_power(np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]]), k)
    m = np.eye(4)
    m[:3, :3] = R
    m[:3, 3] = np.asarray(c) - R @ np.asarray(c)
    return m


def _translate(v):
    m = np.eye(4)
    m[:3, 3] = v
    return m


def _gpu_edit(nf, occ0, lab0, T, dim, ext, moves, lv, pieces=None, rest="keep"):
    occ, lab = occ0.clone(), lab0.clone()
    n = OB.edit_occupancy(nf, T, occ, lab, [(m["label"], m["trans"]) for m in moves], [m["box"] for m in moves], ext, lv, NEAR,
                          FAR, NI, pieces, rest, slab=5000)
    return occ, lab, n


# ---- 1. identity and no-op -------------------------------------------------------------------------------------------------

def test_identity_and_absent_moves_are_bit_exact(nets, golden_dir):
    _, nf, _, _ = nets
    g = np.load(os.path.join(golden_dir, "mesh_grid.npz"))
    T, dim, ext = g["transform_a"], 24, g["extents"]
    occ0, lab0 = _sweep(nf, T, dim, ext)
    lv = _level(occ0)
    o0, l0 = _np(occ0, lab0)
    for mv in _solid_labels(o0, l0, lv, 2):
        occ, lab = OB.edited_sweep(nf, T, [(mv, np.eye(4))], dim, ext, lv, NEAR, FAR, NI)
        assert torch.equal(occ, occ0) and torch.equal(lab, lab0), mv
        cc = OB.object_components(occ0, lab0, lv, 26)
        piece = OB.component_region(cc, [OB.largest_components(cc["label"], cc["voxels"])[mv]], T, ext)
        occ, lab = OB.edited_sweep(nf, T, [(mv, np.eye(4))], dim, ext, lv, NEAR, FAR, NI, pieces=[piece], rest="keep")
        assert torch.equal(occ, occ0) and torch.equal(lab, lab0), mv
    ins_num = int(nf.ins_linear.weight.shape[0]) - 1
    present = set(np.unique(l0[o0 > lv]).tolist())
    absent = [k for k in range(ins_num + 1) if k not in present]
    shift = _translate((0.3, -0.2, 0.1))
    for mv in absent[:1]:
        box = OB.edit_boxes(occ0, lab0, [(mv, shift)], T, ext, lv)[0]
        assert tuple(box) == OB.EMPTY_BOX
        occ, lab, n = _gpu_edit(nf, occ0, lab0, T, dim, ext, [_move(mv, shift, box)], lv)
        assert n == 0 and torch.equal(occ, occ0) and torch.equal(lab, lab0)
    _, _, n = _gpu_edit(nf, occ0, lab0, T, dim, ext, [_move(_solid_labels(o0, l0, lv, 1)[0], shift, OB.EMPTY_BOX)], lv)
    assert n == 0


# ---- 2. exact-grid moves ---------------------------------------------------------------------------------------------------

def _exact_moves(labels, dim):
    labels = [labels[i % len(labels)] for i in range(3)]
    c = np.array([0.125 * 3, -0.125 * 2, 0.0])                        # a grid point of the exact grid
    return [
        _move(labels[0], _translate((0.125 * 3, 0.0, -0.125 * 2)), (4, 28, 3, 29, 5, 27)),
        _move(labels[1], _turn_about(c, 1), (8, 24, 9, 23, 6, 26)),
        _move(labels[2], _translate((-0.25, 0.125, 0.375)) @ _turn_about(c, 2), (0, dim - 1, 10, 20, 0, dim - 1)),
    ]


def test_exact_grid_moves_equal_the_numpy_rule(nets):
    _, nf, _, _ = nets
    T, dim, ext = EXACT["T"], EXACT["dim"], EXACT["ext"]
    occ0, lab0 = _sweep(nf, T, dim, ext)
    lv = _level(occ0)
    o0, l0 = _np(occ0, lab0)
    inv, b = E.grid_index_map(T, ext, dim)
    moves = _exact_moves(_solid_labels(o0, l0, lv), dim)
    for sel in ([0], [1], [2], [0, 1, 2]):
        mv = [moves[i] for i in sel]
        occ, lab, n = _gpu_edit(nf, occ0, lab0, T, dim, ext, mv, lv)
        wo, wl, wn = E.edit(o0, l0, T, ext, mv, E.grid_evaluate(o0, l0, inv, b), lv)
        assert n == wn and n > 0
        np.testing.assert_array_equal(occ.cpu().numpy(), wo)
        np.testing.assert_array_equal(lab.cpu().numpy(), wl)


# ---- 3. off-grid moves against the fp64 network ----------------------------------------------------------------------------

def _fp64_evaluate(wf, ties, near_level, tol, lv):
    p = O.to_torch(wf, torch.float64)

    def f(t):
        x = torch.from_numpy(np.asarray(t, dtype=np.float32)).double()
        raw = O.mlp_forward(p, torch.cat([O.embed(x, 10), O.embed(torch.zeros_like(x), 4)], -1)).numpy()
        occ = 1.0 - np.exp(-np.maximum(raw[:, 3], 0.0) * VOXEL)
        s = 1.0 / (1.0 + np.exp(-raw[:, 4:]))
        top = np.sort(s, 1)
        ties.append(x.numpy()[(top[:, -1] - top[:, -2]) <= 1e-6])
        near_level.append(x.numpy()[np.abs(occ - lv) <= tol])
        return occ, np.argmax(s, 1)
    return f


@pytest.mark.parametrize("mode", ["rotation", "scale", "multi"])
def test_off_grid_moves_agree_with_the_fp64_network(nets, golden_dir, mode):
    _, nf, _, wf = nets
    g = np.load(os.path.join(golden_dir, "mesh_grid.npz"))
    T, dim, ext = g["transform_a"], 16, g["extents"]
    occ0, lab0 = _sweep(nf, T, dim, ext)
    lv = _level(occ0)
    o0, l0 = _np(occ0, lab0)
    mv = _solid_labels(o0, l0, lv, 1)[0]
    A, b = OB.grid_affine(T, dim, ext)
    trans = np.asarray(OB.manipulation_transform(A @ np.full(3, (dim - 1) / 2.0) + b, mode)["transformations"][0]["transformation"])
    box = OB.edit_boxes(occ0, lab0, [(mv, trans)], T, ext, lv)[0]
    occ, lab, n = _gpu_edit(nf, occ0, lab0, T, dim, ext, [_move(mv, trans, box)], lv)
    pts = E.sweep_points(T, ext, dim)
    raw = O.mlp_forward(O.to_torch(wf, torch.float64), torch.cat(
        [O.embed(torch.from_numpy(pts).double(), 10), O.embed(torch.zeros(pts.shape, dtype=torch.float64), 4)], -1)).numpy()
    sig_scale = float(np.abs(raw[:, 3]).max())
    tol = 1e-4 * VOXEL * sig_scale + 2e-6
    ties, near = [], []
    wo, wl, wn = E.edit(o0, l0, T, ext, [_move(mv, trans, box)], _fp64_evaluate(wf, ties, near, tol, lv), lv)
    assert n == wn and n > 0
    go, gl = _np(occ, lab)
    # the target of every grid point, to find the points whose decision rests on an ambiguous network value
    t = E.targets(trans[:3], pts)
    amb_t = {tuple(v) for v in np.concatenate(ties + near)}
    amb = np.array([tuple(v) in amb_t for v in t]).reshape(go.shape)
    differ = (gl != wl) | ((go > lv) != (wo > lv))
    assert not (differ & ~amb).any(), int((differ & ~amb).sum())
    took = (gl == wl) & ~amb
    assert np.abs(go[took].astype(np.float64) - wo[took]).max() <= tol


# ---- 4. the direction of the move -------------------------------------------------------------------------------------------

def test_the_move_carries_the_object_by_the_inverse_transformation(nets):
    _, nf, _, _ = nets
    T, dim, ext = EXACT["T"], EXACT["dim"], EXACT["ext"]
    occ0, lab0 = _sweep(nf, T, dim, ext)
    lv = _level(occ0)
    o0, l0 = _np(occ0, lab0)
    mv = _solid_labels(o0, l0, lv, 1)[0]
    box = (12, 20, 11, 21, 12, 19)
    trans = _translate((0.125 * 3, -0.125, 0.25)) @ _turn_about((0.0, 0.125, 0.0), 1)
    occ, lab, _ = _gpu_edit(nf, occ0, lab0, T, dim, ext, [_move(mv, trans, box)], lv)
    go, gl = _np(occ, lab)
    src = np.zeros(o0.shape, dtype=bool)
    src[box[0]:box[1] + 1, box[2]:box[3] + 1, box[4]:box[5] + 1] = True
    src &= (l0 == mv) & (o0 > lv)
    A, b = OB.grid_affine(T, dim, ext)
    q = np.argwhere(src).astype(np.float64) @ A.T + b                             # source voxels, network frame
    inv_t = np.linalg.inv(trans)
    landed = (q @ inv_t[:3, :3].T + inv_t[:3, 3] - b) @ np.linalg.inv(A).T
    idx = np.rint(landed).astype(np.int64)
    assert np.abs(landed - idx).max() < 1e-9
    want = np.zeros(o0.shape, dtype=bool)
    want[idx[:, 0], idx[:, 1], idx[:, 2]] = True
    np.testing.assert_array_equal((gl == mv) & (go > lv), want)
    inv = OB.inventory_from_grid(occ, lab, T, ext, lv, objects=[mv])
    centre_src = (np.argwhere(src).mean(0)) @ A.T + b
    np.testing.assert_allclose(inv[0]["centre"], inv_t[:3, :3] @ centre_src + inv_t[:3, 3], rtol=0, atol=1e-12)


# ---- 5. pieces ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("rest", ["keep", "drop"])
def test_a_piece_moves_by_the_numpy_rule(nets, rest):
    _, nf, _, _ = nets
    T, dim, ext = EXACT["T"], EXACT["dim"], EXACT["ext"]
    occ0, lab0 = _sweep(nf, T, dim, ext)
    lv = _level(occ0)
    o0, l0 = _np(occ0, lab0)
    cc = OB.object_components(occ0, lab0, lv, 26)
    mv = _solid_labels(o0, l0, lv, 1)[0]
    region = OB.component_region(cc, [OB.largest_components(cc["label"], cc["voxels"])[mv]], T, ext)
    trans = _translate((0.125 * 2, 0.0, -0.125))
    occ, lab = OB.edited_sweep(nf, T, [(mv, trans)], dim, ext, lv, NEAR, FAR, NI, pieces=[region], rest=rest)
    piece = E.Piece(region.bits.cpu().numpy(), dim, region.voxel_map, region.outside == "keep")
    keep = piece.keeps(E.sweep_points(T, ext, dim)).reshape(o0.shape)
    box = E.solid_box(o0, l0, mv, lv, 2, keep)
    assert tuple(OB.edit_boxes(occ0, lab0, [(mv, trans)], T, ext, lv, 2, [region])[0]) == box
    inv, b = E.grid_index_map(T, ext, dim)
    wo, wl, _ = E.edit(o0, l0, T, ext, [_move(mv, trans, box, piece, rest == "drop")], E.grid_evaluate(o0, l0, inv, b), lv)
    np.testing.assert_array_equal(occ.cpu().numpy(), wo)
    np.testing.assert_array_equal(lab.cpu().numpy(), wl)


# ---- 6. the mesh -------------------------------------------------------------------------------------------------------------

def _boundary_plane(p, shape):
    return [(a, x) for a in range(3) for x in (0.0, shape[a] - 1.0) if p[a] == x]


def test_edited_mesh_is_watertight_labelled_by_the_rule_and_reproducible(nets):
    _, nf, _, _ = nets
    T, dim, ext = EXACT["T"], EXACT["dim"], EXACT["ext"]
    occ0, lab0 = _sweep(nf, T, dim, ext)
    lv = _level(occ0)
    mv = _solid_labels(*_np(occ0, lab0), lv, 1)[0]
    moves = [(mv, _translate((0.25, 0.0, -0.125)))]
    runs = [OB.edited_mesh(nf, T, moves, dim, ext, lv, NEAR, FAR, NI, min_cluster=1, per_object=True) for _ in range(2)]
    for k in ("vertices", "triangles", "normals", "clean_vertices", "clean_normals", "clean_triangles", "labels"):
        assert torch.equal(runs[0][k], runs[1][k]), k
    out = runs[0]
    occ, lab = OB.edited_sweep(nf, T, moves, dim, ext, lv, NEAR, FAR, NI)
    v, t = M.marching_cubes(occ, lv)
    assert torch.equal(t, out["triangles"]) and torch.equal(M.to_scene(v, T, dim, ext), out["vertices"])
    v, t = v.cpu().numpy(), t.cpu().numpy()
    directed = np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]])
    _, n_dir = np.unique(directed, axis=0, return_counts=True)
    assert (n_dir == 1).all()
    und, n_und = np.unique(np.sort(directed, 1), axis=0, return_counts=True)
    assert (n_und <= 2).all()
    for a, b in und[n_und == 1]:
        assert set(_boundary_plane(v[a], occ.shape)) & set(_boundary_plane(v[b], occ.shape))
    ci, _, _ = M.clean_mesh(torch.from_numpy(v).to(DEV), None, torch.from_numpy(t).to(DEV), 1)
    o, l = _np(occ, lab)
    want = E.vertex_labels(ci.cpu().numpy(), o, l, lv)
    np.testing.assert_array_equal(out["labels"].cpu().numpy(), want)
    assert (want >= 0).all()
    ins_num = int(nf.ins_linear.weight.shape[0]) - 1
    assert sorted(out["objects"]) == sorted(k for k in np.unique(l[o > lv]).tolist() if k != ins_num)


def test_vertex_labels_kernel_equals_the_rule_on_grid_points():
    lv = 0.45
    g = np.zeros((5, 5, 5), dtype=np.float32)
    labels = np.arange(125, dtype=np.int16).reshape(5, 5, 5)
    g[2, 2, 2] = np.float32(lv)
    for d in [(-1, 0, 0), (1, 0, 0), (0, -1, 0), (0, 1, 0), (0, 0, -1), (0, 0, 1)]:
        g[2 + d[0], 2 + d[1], 2 + d[2]] = 0.9
    v, _ = M.marching_cubes(torch.from_numpy(g).to(DEV), lv)
    extra = torch.tensor([[1.0, 2.0, 2.0], [9.0, 9.0, 9.0], [float("nan"), 0.0, 0.0], [-1.5, 2.0, 2.0]], device=DEV)
    v = torch.cat([v, extra])
    got = M.vertex_labels(v, torch.from_numpy(g).to(DEV), torch.from_numpy(labels).to(DEV), lv).cpu().numpy()
    np.testing.assert_array_equal(got, E.vertex_labels(v.cpu().numpy(), g, labels, lv))
    assert (got[np.all(v.cpu().numpy() == 2.0, axis=1)] == labels[1, 2, 2]).all()


def test_move_objects_writes_the_edited_meshes(tmp_path):
    nc, nf, _, _ = make_models(7, 8, 13, "cpu", trained_like=True)
    torch.save({"network_coarse_state_dict": nc.state_dict(), "network_fine_state_dict": nf.state_dict()}, tmp_path / "ck.tar")
    np.save(tmp_path / "T.npy", np.eye(4))
    pose = np.eye(4, dtype=np.float32)
    pose[2, 3] = 6.0
    np.save(tmp_path / "pose.npy", pose)
    # the label with the most solid points in the tool's own sweep (every label but the last)
    _, nf_d, _, _ = make_models(7, 8, 13, DEV, trained_like=True)
    o, l = _np(*OB.occupancy_objects(nf_d, np.eye(4), OB.object_mask(13, keep=range(13)), 32, (1.9, 7.0, 7.0), device=DEV))
    lv = _level(torch.from_numpy(o))
    label = _solid_labels(o, l, lv, 1)[0]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "move_objects.py"), str(tmp_path / "ck.tar"), "--pose",
                        str(tmp_path / "pose.npy"), "--hwk", "24", "32", "30", "0", "16", "0", "30", "12", "0", "0", "1",
                        "--move-label", str(label), "--mode", "translation", "--transform", str(tmp_path / "T.npy"),
                        "--grid-dim", "32", "--level", repr(lv), "--out", str(tmp_path / "o"), "--mesh", "--min-cluster", "1",
                        "--N-test", "256"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    info = json.loads(r.stdout.strip().splitlines()[-1])
    assert {"rgb.png", "instance.png", "edited.ply", "color_edited.ply"} <= set(info["files"])
    a, b = M.read_ply(tmp_path / "o" / "edited.ply"), M.read_ply(tmp_path / "o" / "color_edited.ply")
    assert (len(a["vertices"]), len(a["faces"])) == (info["mesh"]["vertices"], info["mesh"]["triangles"])
    assert len(b["vertices"]) == info["mesh"]["clean_vertices"] and b["colors"] is not None and len(a["faces"]) > 0


# ---- 7. rejections -----------------------------------------------------------------------------------------------------------

def test_the_library_rejects_bad_moves(nets):
    lv = 0.45
    _, nf, _, _ = nets
    ins_num = int(nf.ins_linear.weight.shape[0]) - 1
    ctx = get_context(DEV)
    slot = ctx.slot_for(nf)
    ctx.bind(slot, nf)
    dim = 8
    occ = torch.zeros((dim,) * 3, device=DEV)
    lab = torch.zeros((dim,) * 3, device=DEV, dtype=torch.int16)
    cc = OB.object_components(occ + 1.0, lab, lv, 26)
    region = OB.component_region(cc, [0], np.eye(4), (4.0, 4.0, 4.0))             # applies to label 0 only

    def call(moves, level=lv):
        arr = (_lib.EditMove * max(1, len(moves)))()
        for i, m in enumerate(moves):
            arr[i].label, arr[i].rest_drop = m.get("label", 1), 0
            arr[i].trans[:] = list(np.asarray(m.get("trans", np.eye(4)), dtype=np.float64)[:3].reshape(-1))
            arr[i].box[:] = list(m.get("box", (0, dim - 1) * 3))
            if "piece" in m:
                arr[i].piece = m["piece"]
        n = C.c_int64(-1)
        with pytest.raises(RuntimeError) as e:
            ctx.call("dmnerf_mesh_occupancy_edit", ctx.handle, slot, _lib.doubles(np.eye(4), 16), _lib.doubles((4.0, 4.0, 4.0), 3), dim,
                     VOXEL, level, 0, arr, len(moves), _lib.ptr(occ), _lib.ptr(lab, torch.int16), C.byref(n))
        return str(e.value)

    assert "between 0 and 8" in call([{}] * 9)
    assert "outside [0, %d]" % ins_num in call([{"label": ins_num + 1}])
    assert "outside [0, %d]" % ins_num in call([{"label": -1}])
    assert "not finite" in call([{"trans": np.full((4, 4), np.inf)}])
    assert "det" in call([{"trans": np.diag([1.0, -1.0, 1.0, 1.0])}])
    assert "det" in call([{"trans": np.zeros((4, 4))}])
    assert "inverted or outside" in call([{"box": (0, dim, 0, 1, 0, 1)}])
    assert "inverted or outside" in call([{"box": (3, 2, 0, 1, 0, 1)}])
    assert "inverted or outside" in call([{"box": (-1, 2, 0, 1, 0, 1)}])
    assert "level" in call([{}], level=1.0)
    assert "level" in call([{}], level=0.0)
    assert "applies to" in call([{"label": 1, "piece": region.abi(ins_num)}])
    assert torch.count_nonzero(occ) == 0 and torch.count_nonzero(lab) == 0
    with pytest.raises(ValueError, match="outside"):
        OB.edited_sweep(nf, np.eye(4), [(ins_num + 1, np.eye(4))], dim, (4.0, 4.0, 4.0))
    with pytest.raises(ValueError, match="applies to"):
        OB.edited_sweep(nf, np.eye(4), [(1, np.eye(4))], dim, (4.0, 4.0, 4.0), pieces=[region])
