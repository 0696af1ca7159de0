"""GPU: grid_view(moves=, source=) and dmnerf_grid_edit_source against oracle/edit_view_oracle.py on seeded keep-all sweeps
(ins_num 13 and 93): the move, the colour point and the direction bit for bit for edited_grid's whole-voxel translation, quarter
turn, manipulation_transform rotation and scale, two moves, a piece with the rest kept and dropped, a copy, a group, each
deformation kind and an arrange_objects result; the colour against the network at the oracle's point and direction (exact and
fp16), and against grid_view without moves off the moved pixels; the identity move; the consistency check on the source and on
an edited_sweep grid, before the network runs; repeats and view batches; the host rejections; and move_objects.py --preview."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from dmnerf_b200 import _lib, synth
from dmnerf_b200 import objects as OB
from dmnerf_b200.autograd import mlp_forward_points
from dmnerf_b200.engine import get_context
from dmnerf_b200.helpers import get_rays_k
from dmnerf_b200.testing import make_models
from oracle import edit_sweep_oracle as E
from oracle import edit_view_oracle as EV

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
NI = 128
DIM = 64
EXT = (4.0, 4.0, 4.0)
T = np.eye(4)
H, W = 48, 64
UP = np.array([0.0, 0.0, 1.0])
DOWN = (0.0, 0.0, -1.0)


@pytest.fixture(scope="module", params=[13, 93])
def scene(request):
    nc, nf, _, _ = make_models(101, 202, request.param, DEV)
    wl = synth.workload("dmsr_study")
    with torch.no_grad():
        occ, lab = OB.occupancy_objects(nf, T, OB.object_mask(request.param, remove=[]), DIM, EXT, wl["near"], wl["far"], NI,
                                        device=DEV)
    x = occ.flatten()
    x = x[x > 0]
    level = float(x.kthvalue(max(1, int(0.5 * x.numel()))).values)
    # the synthetic network may label its whole sweep with one object: split every label into the four horizontal quadrants of
    # the grid (index axes i and k; j is up), so that the moves below have several objects side by side to move, copy, carry
    # and overwrite.  The edits are grid-only, so the labels need not be the network's.
    i = torch.arange(DIM, device=DEV)
    quad = (2 * (i[:, None, None] >= DIM // 2) + (i[None, None, :] >= DIM // 2)).to(torch.int16)
    lab_net = lab
    lab = ((lab_net % 32) * 4 + quad).to(torch.int16).contiguous()
    o, l = occ.cpu().numpy(), lab.cpu().numpy()
    by_size = _by_size(o, l, level)
    assert len(by_size) >= 2, "the quadrants of the sweep hold fewer than two objects"
    K = np.asarray(wl["K"], dtype=np.float32).copy()
    K[0] *= W / wl["W"]
    K[1] *= H / wl["H"]
    c2w = np.eye(4, dtype=np.float32)
    c2w[:3] = np.asarray(wl["c2w"], dtype=np.float32)[:3]
    return dict(nc=nc, nf=nf, occ=occ, lab=lab, o=o, l=l, level=level, ins_num=request.param, by_size=by_size, K=K, c2w=c2w,
                near=float(wl["near"]), far=float(wl["far"]), lab_net=lab_net,
                by_size_net=_by_size(o, lab_net.cpu().numpy(), level))


def _by_size(o, l, level):
    """The labels with solid points, most points first."""
    k, cnt = np.unique(l[o > np.float32(level)], return_counts=True)
    return [int(v) for v in k[np.argsort(-cnt, kind="stable")]]


def _centre(s, label):
    A, b = OB.grid_affine(T, DIM, EXT)
    idx = np.argwhere((s["l"] == label) & (s["o"] > np.float32(s["level"])))
    return A @ idx.mean(0) + b, (idx @ A.T + b)


def _translate(delta):
    A, _ = OB.grid_affine(T, DIM, EXT)
    m = np.eye(4)
    m[:3, 3] = A @ np.asarray(delta, dtype=np.float64)
    return m


def _half_piece(s, label, axis=0):
    """The half of `label`'s solid points below its median index along `axis`, as a Region that applies to `label`."""
    idx = np.argwhere((s["l"] == label) & (s["o"] > np.float32(s["level"])))
    cut = int(np.median(idx[:, axis]))
    mask = torch.zeros((DIM,) * 3, dtype=torch.bool, device=DEV)
    sl = [slice(None)] * 3
    sl[axis] = slice(0, cut + 1)
    mask[tuple(sl)] = True
    return OB.region_from_mask(mask, T, EXT, applies=[label], outside="drop")


def _deformation(s, label, kind):
    c, pts = _centre(s, label)
    h = (pts - c) @ UP
    kw = {"twist": dict(twist=lambda u: 50.0 * u), "bend": dict(bend=lambda u: 0.2 * u * u, bend_dir=(1.0, 0.0, 0.0)),
          "taper": dict(taper=lambda u: 1.0 - 0.3 * u)}[kind]
    return OB.deformation(c, UP, float(h.min()) - 0.05, float(h.max()) + 0.05, 17, **kw)


def _case(s, name):
    """(moves, edit keywords, the grid they give) of a named case, or None where the synthetic sweep cannot make it."""
    big, second = s["by_size"][0], s["by_size"][1]
    kw = {}
    if name == "translation":
        moves = [(big, _translate((3, 0, -2)))]
    elif name == "quarter_turn":
        moves = [(big, OB.manipulation_transform(_centre(s, big)[0], "rotation", yaw=90.0)["transformations"][0]["transformation"])]
    elif name in ("rotation", "scale"):
        moves = [(big, OB.manipulation_transform(_centre(s, big)[0], name, yaw=30.0)["transformations"][0]["transformation"])]
    elif name == "two_moves":
        moves = [(big, _translate((4, 0, 0))), (second, _translate((-3, 2, 0)))]
    elif name in ("piece_keep", "piece_drop"):
        moves = [(big, _translate((5, 0, 0)))]
        kw = dict(pieces=[_half_piece(s, big)], rest="keep" if name == "piece_keep" else "drop")
    elif name == "copy":
        moves = [(second, _translate((0, 6, 0)))]
        kw = dict(copies=[True])
    elif name == "group":
        group = sorted(set(OB.carried_labels(s["occ"], s["lab"], T, big, DOWN, EXT, s["level"])["group"]) | {big, second})
        moves = [(big, _translate((4, 0, 2)))]
        kw = dict(groups=[group])
    elif name in ("twist", "bend", "taper"):
        moves = [(big, _translate((2, 0, 0)))]
        kw = dict(deformations=[_deformation(s, big, name)])
    elif name == "arrange":
        A, b = OB.grid_affine(T, DIM, EXT)
        items = [{"label": second, "near": (A @ np.array([DIM / 2, DIM / 2, DIM / 4]) + b).tolist(), "turns": 4, "stable": False}]
        r = OB.arrange_objects(s["occ"], s["lab"], T, items, DOWN, EXT, s["level"])
        if not r["moves"]:
            return None
        return r["moves"], dict(pieces=r["pieces"], rest=r["rest"], copies=r["copies"], groups=r["groups"]), (r["occ"], r["labels"])
    e_occ, e_lab, _ = OB.edited_grid(s["occ"], s["lab"], T, moves, EXT, s["level"], **kw)
    return moves, kw, (e_occ, e_lab)


def _oracle_moves(s, moves, moved, kw):
    pieces = kw.get("pieces") or [None] * len(moves)
    out = []
    for i, (label, trans) in enumerate(moves):
        p = pieces[i]
        mv = dict(label=label, trans=np.asarray(trans, dtype=np.float64), box=moved.boxes[i], rest_drop=moved.rest_drop[i],
                  copy=moved.copies[i], group=list(moved.groups[i]), deform=moved.deformations[i])
        if p is not None:
            mv["piece"] = E.Piece(p.bits.cpu().numpy(), p.dim, p.voxel_map, p.outside == "keep")
            mv["applies"] = OB.kept_labels(p.applies_words(s["ins_num"]))
        out.append(mv)
    return out


def _rays(s, poses):
    pose = torch.as_tensor(poses, dtype=torch.float32, device=DEV)
    pose = pose[None] if pose.dim() == 2 else pose
    rays = [get_rays_k(H, W, s["K"], pose[v]) for v in range(pose.shape[0])]
    return torch.stack([r[0] for r in rays]), torch.stack([r[1] for r in rays])


def _moved(s, moves, kw):
    return OB.render_moves(s["occ"], s["lab"], T, moves, EXT, s["level"], s["near"], s["far"], NI, **kw)


CASES = ["translation", "quarter_turn", "rotation", "scale", "two_moves", "piece_keep", "piece_drop", "copy", "group", "twist",
         "bend", "taper", "arrange"]


@pytest.mark.parametrize("name", CASES)
def test_provenance_point_and_direction_equal_the_oracle(scene, name):
    s = scene
    case = _case(s, name)
    if case is None:
        pytest.skip("the synthetic sweep cannot place this case")
    moves, kw, (e_occ, e_lab) = case
    moved = _moved(s, moves, kw)
    o, d = _rays(s, s["c2w"])
    c = OB.cast_grid(e_occ, e_lab, T, o, d, s["near"], s["far"], EXT, s["level"])
    move, point, vdir = OB._edit_view(e_occ, e_lab, moved, (s["occ"], s["lab"]), o, d, c)
    dim = DIM
    vox = c["voxel"].reshape(-1, 3).cpu().numpy().astype(np.int64)
    lin = np.where(vox[:, 0] >= 0, (vox[:, 0] * dim + vox[:, 1]) * dim + vox[:, 2], -1)
    om = _oracle_moves(s, moves, moved, kw)
    m_ref, occ_r, lab_r = EV.provenance(s["o"], s["l"], T, EXT, om, lin, s["level"])
    assert not EV.mismatched(e_occ.cpu().numpy(), e_lab.cpu().numpy(), lin, occ_r, lab_r).any()
    p_ref, d_ref = EV.colour_rays(o.cpu().numpy(), d.cpu().numpy(), c["depth"].reshape(-1).cpu().numpy(), lin, m_ref, om)
    assert np.array_equal(move.reshape(-1).cpu().numpy(), m_ref)
    assert np.array_equal(point.reshape(-1, 3).cpu().numpy().view(np.int32), p_ref.view(np.int32))
    assert np.array_equal(vdir.reshape(-1, 3).cpu().numpy().view(np.int32), d_ref.view(np.int32))
    assert (m_ref >= 0).sum() > 0, "no hit pixel shows a moved object"


@pytest.mark.parametrize("f16", [False, True])
@pytest.mark.parametrize("name", ["translation", "rotation", "two_moves", "piece_keep", "copy", "twist"])
def test_colour_is_the_network_at_the_source(scene, name, f16, monkeypatch):
    if f16:
        monkeypatch.setattr(_lib, "INFER_IMPL", _lib.IMPL_UMMA_F16)
    s = scene
    moves, kw, (e_occ, e_lab) = _case(s, name)
    moved = _moved(s, moves, kw)
    args = (e_occ, e_lab, T, H, W, s["K"], torch.from_numpy(s["c2w"]).to(DEV), s["near"], s["far"], EXT, s["level"])
    view = OB.grid_view(*args, model_fine=s["nf"], moves=moved, source=(s["occ"], s["lab"]))
    plain = OB.grid_view(*args, model_fine=s["nf"])
    o, d = _rays(s, s["c2w"])
    c = OB.cast_grid(e_occ, e_lab, T, o, d, s["near"], s["far"], EXT, s["level"])
    move, point, vdir = OB._edit_view(e_occ, e_lab, moved, (s["occ"], s["lab"]), o, d, c)
    hit, mv = c["hit"][0], view["move"]
    movedpx = mv >= 0
    assert torch.equal(mv, move[0]) and movedpx.any() and (mv[~hit] == -1).all()
    pts = torch.where(movedpx[..., None], point[0], c["point"][0])
    dirs = d[0] / torch.norm(d[0], dim=-1, keepdim=True)
    vd = torch.where(movedpx[..., None], vdir[0] / torch.norm(vdir[0], dim=-1, keepdim=True), dirs)
    with torch.no_grad():
        ref = torch.sigmoid(mlp_forward_points(s["nf"], pts[hit], vd[hit])[:, :3])
    assert torch.equal(view["rgb"][hit], ref)
    still = hit & ~movedpx
    assert torch.equal(view["rgb"][still], plain["rgb"][still])
    assert (view["rgb"][~hit] == 0).all()
    for key in ("depth", "label", "normal", "hit"):
        assert torch.equal(view[key], plain[key]), key


@pytest.mark.parametrize("with_piece", [False, True])
def test_identity_move_gives_todays_colours(scene, with_piece):
    s = scene
    big = s["by_size"][0]
    kw = dict(pieces=[_half_piece(s, big)]) if with_piece else {}
    moves = [(big, np.eye(4))]
    e_occ, e_lab, _ = OB.edited_grid(s["occ"], s["lab"], T, moves, EXT, s["level"], **kw)
    assert torch.equal(e_occ, s["occ"]) and torch.equal(e_lab, s["lab"])
    moved = _moved(s, moves, kw)
    args = (e_occ, e_lab, T, H, W, s["K"], torch.from_numpy(s["c2w"]).to(DEV), s["near"], s["far"], EXT, s["level"])
    view = OB.grid_view(*args, model_fine=s["nf"], moves=moved, source=(s["occ"], s["lab"]))
    plain = OB.grid_view(*args, model_fine=s["nf"])
    assert torch.equal(view["rgb"], plain["rgb"])
    if not with_piece:
        assert torch.equal(view["move"] == 0, view["hit"] & (view["label"] == big))
    else:
        assert (view["move"][view["move"] >= 0] == 0).all() and (view["label"][view["move"] == 0] == big).all()
    # the source tensors themselves viewed as their own identity edit
    same = OB.grid_view(s["occ"], s["lab"], *args[2:], model_fine=s["nf"], moves=moved, source=(s["occ"], s["lab"]))
    assert torch.equal(same["rgb"], plain["rgb"]) and torch.equal(same["move"], view["move"])


def test_a_grid_that_is_not_the_edit_raises_before_the_network(scene, monkeypatch):
    # edited_sweep evaluates the network, so this case moves the network's own largest label on the network's labels
    s = dict(scene, lab=scene["lab_net"], l=scene["lab_net"].cpu().numpy())
    moves = [(s["by_size_net"][0], _translate((3, 0, -2)))]
    moved = _moved(s, moves, {})
    calls = []
    import dmnerf_b200.autograd as AG
    real = AG.mlp_forward_points
    monkeypatch.setattr(AG, "mlp_forward_points", lambda *a, **k: calls.append(1) or real(*a, **k))
    args = (T, H, W, s["K"], torch.from_numpy(s["c2w"]).to(DEV), s["near"], s["far"], EXT, s["level"])
    with pytest.raises(ValueError, match=r"grid_view: \d+ of \d+ hit voxels differ"):
        OB.grid_view(s["occ"], s["lab"], *args, model_fine=s["nf"], moves=moved, source=(s["occ"], s["lab"]))
    with torch.no_grad():
        sw_occ, sw_lab = OB.edited_sweep(s["nf"], T, moves, DIM, EXT, s["level"], s["near"], s["far"], NI)[:2]
    e_occ, e_lab, _ = OB.edited_grid(s["occ"], s["lab"], T, moves, EXT, s["level"])
    o, d = _rays(s, s["c2w"])
    c = OB.cast_grid(sw_occ, sw_lab, T, o, d, s["near"], s["far"], EXT, s["level"])
    v = c["voxel"][c["hit"]]
    differ = (sw_occ[v[:, 0], v[:, 1], v[:, 2]] != e_occ[v[:, 0], v[:, 1], v[:, 2]]) | \
             (sw_lab[v[:, 0], v[:, 1], v[:, 2]] != e_lab[v[:, 0], v[:, 1], v[:, 2]])
    if bool(differ.any()):
        with pytest.raises(ValueError, match="hit voxels differ"):
            OB.grid_view(sw_occ, sw_lab, *args, model_fine=s["nf"], moves=moved, source=(s["occ"], s["lab"]))
    assert not calls


def test_repeats_are_bit_identical_and_batches_equal_single_views(scene):
    s = scene
    moves, kw, (e_occ, e_lab) = _case(s, "two_moves")
    moved = _moved(s, moves, kw)
    poses = np.stack([s["c2w"], synth.pose_spherical(30.0, -20.0, 4.0), synth.pose_spherical(-70.0, -35.0, 3.5)]).astype(np.float32)
    args = (e_occ, e_lab, T, H, W, s["K"])
    rest = (s["near"], s["far"], EXT, s["level"])
    batch = OB.grid_view(*args, torch.from_numpy(poses).to(DEV), *rest, model_fine=s["nf"], moves=moved, source=(s["occ"], s["lab"]))
    again = OB.grid_view(*args, torch.from_numpy(poses).to(DEV), *rest, model_fine=s["nf"], moves=moved, source=(s["occ"], s["lab"]))
    for key in ("move", "rgb", "depth", "label"):
        assert torch.equal(batch[key], again[key]), key
    for v in range(3):
        one = OB.grid_view(*args, torch.from_numpy(poses[v]).to(DEV), *rest, model_fine=s["nf"], moves=moved,
                           source=(s["occ"], s["lab"]))
        assert torch.equal(batch["move"][v], one["move"])
        # the network may take another kernel for another number of points: the colours agree to its rounding
        assert torch.allclose(batch["rgb"][v], one["rgb"], atol=1e-5, rtol=0)


def test_rejections_name_the_entry_point(scene):
    s = scene
    moves, kw, (e_occ, e_lab) = _case(s, "translation")
    moved = _moved(s, moves, kw)
    n = 16
    o = torch.zeros((n, 3), device=DEV)
    d = torch.ones((n, 3), device=DEV)
    t = torch.ones(n, device=DEV)
    vox = torch.full((n,), -1, dtype=torch.int32, device=DEV)
    mo = torch.full((n,), 7, dtype=torch.int32, device=DEV)
    pt = torch.full((n, 3), 7.0, device=DEV)
    dr = torch.full((n, 3), 7.0, device=DEV)
    ctx = get_context(DEV)
    mism = ctypes.c_int64(0)
    good = dict(occ=_lib.ptr(e_occ), lab=_lib.ptr(e_lab, torch.int16), socc=_lib.ptr(s["occ"]), slab=_lib.ptr(s["lab"], torch.int16),
                moves=ctypes.byref(moved.abi()), o=_lib.ptr(o), d=_lib.ptr(d), t=_lib.ptr(t), vox=_lib.ptr(vox, torch.int32), n=n,
                mo=_lib.ptr(mo, torch.int32), pt=_lib.ptr(pt), dr=_lib.ptr(dr), mism=ctypes.byref(mism))

    def call(a, handle=ctx.handle):
        ctx.call("dmnerf_grid_edit_source", handle, a["occ"], a["lab"], a["socc"], a["slab"], a["moves"], None, None, None, a["o"],
                 a["d"], a["t"], a["vox"], a["n"], a["mo"], a["pt"], a["dr"], a["mism"])
    call(good)
    assert mism.value == 0 and (mo == -1).all() and torch.isnan(pt).all() and (dr == 0).all()
    bad_move = _lib.EditMove.from_buffer_copy(moved.abi().moves[0])
    bad_move.label = 128
    desc = _lib.RenderMoves.from_buffer_copy(moved.abi())
    desc.moves = ctypes.pointer(bad_move)
    empty = _lib.RenderMoves.from_buffer_copy(moved.abi())
    empty.n_moves = 0
    flat = _lib.RenderMoves.from_buffer_copy(moved.abi())
    flat.level = 1.5
    for change in (dict(occ=None), dict(slab=None), dict(moves=None), dict(n=-1), dict(o=None), dict(mo=None), dict(mism=None),
                   dict(socc=_lib.ptr(e_occ)), dict(moves=ctypes.byref(desc)), dict(moves=ctypes.byref(empty)),
                   dict(moves=ctypes.byref(flat))):
        with pytest.raises(RuntimeError, match="grid_edit_source"):
            call(dict(good, **change))
    with pytest.raises(RuntimeError, match="grid_edit_source: ctx is NULL"):
        call(good, None)
    vox.fill_(DIM ** 3)
    with pytest.raises(RuntimeError, match="grid_edit_source: .* voxel indices outside"):
        call(good)


@pytest.mark.parametrize("extra", [[], ["--copy"], ["--twist", "30", "--up", "0", "0", "1"]])
def test_move_objects_preview_writes_the_edited_colour(scene, tmp_path, extra):
    s = scene
    nc, nf = s["nc"], s["nf"]
    ck = tmp_path / "ck.tar"
    torch.save({"network_coarse_state_dict": {k: v.cpu() for k, v in nc.state_dict().items()},
                "network_fine_state_dict": {k: v.cpu() for k, v in nf.state_dict().items()}}, str(ck))
    wl = synth.workload("dmsr_study")
    K = np.asarray(wl["K"], dtype=np.float64).copy()
    K[0] *= 8 / wl["W"]
    K[1] *= 8 / wl["H"]
    np.save(str(tmp_path / "pose.npy"), s["c2w"])
    np.save(str(tmp_path / "T.npy"), T)
    out = tmp_path / "out"
    cmd = [sys.executable, os.path.join(ROOT, "tools", "move_objects.py"), str(ck), "--pose", str(tmp_path / "pose.npy"), "--hwk",
           "8", "8", *map(str, K.reshape(-1)), "--transform", str(tmp_path / "T.npy"), "--extents", *map(str, EXT),
           "--grid-dim", str(DIM), "--level", str(s["level"]), "--near", str(wl["near"]), "--far", str(wl["far"]), "--move-label",
           str(s["by_size_net"][0]), "--mode", "translation", "--distance", "0.25", "--preview", "--render", "none", "--out", str(out),
           *extra]
    p = subprocess.run(cmd, capture_output=True, text=True, cwd=str(tmp_path))
    assert p.returncode == 0, p.stderr[-3000:]
    rec = json.loads(p.stdout.strip().splitlines()[-1])
    assert {"preview.png", "preview_edited.png", "preview_rgb.png", "preview_edited_rgb.png"} <= set(rec["files"])
    assert os.path.getsize(os.path.join(str(out), "preview_edited_rgb.png")) > 0
