"""GPU: dmnerf_grid_cast, cast_grid and grid_view against the flat walk of oracle/grid_cast_oracle.py: depth, label and voxel bit
for bit and normals to 1e-5, on analytic grids at dims 2, 3, 17, 64 and 256, seeded keep-all sweeps
and an edited_grid of one, with the synth frames' rays and random rays from inside, outside and along the axes; the keep mask, the
repeat, grid_view against cast_grid, the network colour, the picked piece, the rejections and tools/move_objects.py --pick."""
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
from dmnerf_b200.helpers import get_rays_at, get_rays_k
from dmnerf_b200.testing import make_models
from oracle import edit_sweep_oracle as E
from oracle import grid_cast_oracle as G

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
NI = 128
EXT = (4.0, 4.0, 4.0)
A = 0.6
T_ROT = np.array([[np.cos(A), 0.0, np.sin(A), 0.1], [0.0, 1.0, 0.0, -0.2], [-np.sin(A), 0.0, np.cos(A), 0.15], [0, 0, 0, 1.0]])


def _analytic(kind, dim, seed=0):
    rng = np.random.default_rng(seed + dim)
    idx = np.indices((dim,) * 3).transpose(1, 2, 3, 0).astype(np.float64)
    c = (dim - 1) / 2.0
    if kind == "sphere":
        r = np.linalg.norm(idx - c - 0.3, axis=-1)
        occ = np.clip(0.5 + (0.35 * dim - r) / 2.0, 0, 1)
        lab = (idx[..., 0] > c).astype(np.int16) + 3
    elif kind == "boxes":
        occ = np.zeros((dim,) * 3)
        lab = np.zeros((dim,) * 3, dtype=np.int16)
        for b in range(6):
            lo = rng.integers(0, dim, 3)
            hi = np.minimum(lo + rng.integers(0, max(2, dim // 3), 3), dim - 1)
            occ[lo[0]:hi[0] + 1, lo[1]:hi[1] + 1, lo[2]:hi[2] + 1] = rng.uniform(0.5, 1.0)
            lab[lo[0]:hi[0] + 1, lo[1]:hi[1] + 1, lo[2]:hi[2] + 1] = b + 1
    else:                                                         # scattered points: long walks through empty space
        occ = (rng.random((dim,) * 3) < 2.0 / dim).astype(np.float64) * rng.uniform(0.46, 1.0, (dim,) * 3)
        lab = rng.integers(0, 20, (dim,) * 3).astype(np.int16)
    return occ.astype(np.float32), lab


def _rays(dim, T, ext, n, seed):
    """Random rays from outside, from inside and along the grid's index axes (network frame, fp32)."""
    rng = np.random.default_rng(seed)
    inv, b = E.grid_index_map(T, ext, dim)
    M = np.linalg.inv(inv)
    to_net = lambda u: (u @ M.T + b).astype(np.float32)             # noqa: E731
    dir_net = lambda u: (u @ M.T).astype(np.float32)                 # noqa: E731
    k = n // 4
    c = (dim - 1) / 2.0
    u_out = c + rng.normal(size=(k, 3)) * 2 * dim
    aim = rng.uniform(-0.5, dim - 0.5, (k, 3))
    u_in = rng.uniform(-0.5, dim - 0.5, (k, 3))
    d_in = rng.normal(size=(k, 3))
    axes = np.eye(3)[rng.integers(0, 3, k)] * rng.choice([-1.0, 1.0], (k, 1))
    u_ax = rng.integers(0, dim, (k, 3)).astype(np.float64) + rng.choice([0.0, 0.5, 0.25], (k, 3))
    u_ax = u_ax - axes * (dim + 2)                                    # outside, heading in
    corner = rng.integers(0, dim, (n - 3 * k, 3)) - 0.5
    d_c = rng.integers(-2, 3, (n - 3 * k, 3)).astype(np.float64)
    o = np.concatenate([to_net(u_out), to_net(u_in), to_net(u_ax), to_net(corner)])
    d = np.concatenate([dir_net(aim - u_out), dir_net(d_in), dir_net(axes), dir_net(d_c)])
    return o, d


def _check(occ, lab, T, ext, o, d, near, far, level=0.45, keep=None, remove=None, normals=True):
    occ_d = torch.from_numpy(occ).to(DEV)
    lab_d = torch.from_numpy(lab).to(DEV)
    r = OB.cast_grid(occ_d, lab_d, T, torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), near, far, ext, level, keep, remove,
                     normals=normals)
    words = OB._cast_words(keep, remove)
    ref = G.cast(occ, lab, T, ext, o, d, near, far, level, words)
    dim = occ.shape[0]
    vox = r["voxel"].cpu().numpy()
    lin = np.where(vox[:, 0] >= 0, (vox[:, 0] * dim + vox[:, 1]) * dim + vox[:, 2], -1)
    assert np.array_equal(lin, ref["voxel"]), np.nonzero(lin != ref["voxel"])[0][:10]
    assert np.array_equal(r["depth"].cpu().numpy().view(np.int32), ref["t"].view(np.int32))
    assert np.array_equal(r["label"].cpu().numpy(), ref["label"])
    assert np.array_equal(r["hit"].cpu().numpy(), ref["voxel"] >= 0)
    if normals:
        assert np.abs(r["normal"].cpu().numpy().astype(np.float64) - ref["normal"]).max() <= 1e-5
    return r, ref


@pytest.mark.parametrize("dim", [2, 3, 17, 64, 256])
@pytest.mark.parametrize("kind", ["sphere", "boxes", "scatter"])
def test_analytic_grids_equal_the_flat_walk(kind, dim):
    occ, lab = _analytic(kind, dim)
    for T, ext in ((np.eye(4), (dim - 1.0,) * 3), (T_ROT, (1.9, 7.0, 4.0))):
        o, d = _rays(dim, T, ext, 4096 if dim < 256 else 2048, dim)
        r, ref = _check(occ, lab, T, ext, o, d, 0.0, 1e4)
        assert (ref["voxel"] >= 0).sum() > 0.05 * len(o)
        _check(occ, lab, T, ext, o, d, 0.7, 0.7 + float(np.max(ext)))     # clipped by near and far


@pytest.fixture(scope="module", params=[13, 93])
def scene(request):
    nc, nf, _, _ = make_models(101, 202, request.param, DEV)
    wl = synth.workload("dmsr_study")
    with torch.no_grad():
        occ, lab = OB.occupancy_objects(nf, np.eye(4), OB.object_mask(request.param, remove=[]), 64, EXT, wl["near"], wl["far"], NI,
                                        device=DEV)
    x = occ.flatten()
    x = x[x > 0]
    level = float(x.kthvalue(max(1, int(0.5 * x.numel()))).values)
    return dict(nc=nc, nf=nf, occ=occ, lab=lab, level=level, ins_num=request.param)


def _frame_rays(name, n=8192):
    wl = synth.workload(name)
    sel = np.linspace(0, wl["H"] * wl["W"] - 1, n).astype(np.int64)
    return wl["rays_o"][sel].astype(np.float32), wl["rays_d"][sel].astype(np.float32), wl["near"], wl["far"]


@pytest.mark.parametrize("frames", ["dmsr_study", "replica_room0_93"])
def test_sweeps_and_edited_grid_equal_the_flat_walk(scene, frames):
    occ, lab = scene["occ"].cpu().numpy(), scene["lab"].cpu().numpy()
    o, d, near, far = _frame_rays(frames)
    ro, rd = _rays(occ.shape[0], np.eye(4), EXT, 2048, 7)
    o, d = np.concatenate([o, ro]), np.concatenate([d, rd])
    r, ref = _check(occ, lab, np.eye(4), EXT, o, d, near, far, scene["level"])
    assert (ref["voxel"] >= 0).sum() > 100
    # one move of the largest label by whole voxels (0.125 network units per voxel here: 64 - 1 steps over 4)
    k, cnt = np.unique(lab[occ > np.float32(scene["level"])], return_counts=True)
    mv = int(k[np.argmax(cnt)])
    trans = np.eye(4)
    trans[:3, 3] = (0.25, 0.0, -0.125)
    e_occ, e_lab, _ = OB.edited_grid(scene["occ"], scene["lab"], np.eye(4), [(mv, trans)], EXT, scene["level"])
    _check(e_occ.cpu().numpy(), e_lab.cpu().numpy(), np.eye(4), EXT, o, d, near, far, scene["level"])


def test_keep_and_remove_equal_a_grid_without_the_other_labels(scene):
    occ, lab = scene["occ"].cpu().numpy(), scene["lab"].cpu().numpy()
    o, d, near, far = _frame_rays("dmsr_study", 4096)
    present = np.unique(lab[occ > np.float32(scene["level"])])
    keep = [int(v) for v in present[::2]]
    for kw, kept in ((dict(keep=keep), np.isin(lab, keep)), (dict(remove=keep), ~np.isin(lab, keep))):
        r, _ = _check(occ, lab, np.eye(4), EXT, o, d, near, far, scene["level"], normals=False, **kw)
        bare = OB.cast_grid(torch.from_numpy(np.where(kept, occ, 0).astype(np.float32)).to(DEV), scene["lab"], np.eye(4),
                            torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), near, far, EXT, scene["level"], normals=False)
        for key in ("depth", "label", "voxel", "hit"):
            assert torch.equal(r[key], bare[key]), key


def test_repeated_calls_are_bit_identical(scene):
    o, d, near, far = _frame_rays("replica_room0_93")
    o, d = torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV)
    runs = [OB.cast_grid(scene["occ"], scene["lab"], np.eye(4), o, d, near, far, EXT, scene["level"]) for _ in range(3)]
    for r in runs[1:]:
        for key in ("depth", "label", "voxel", "normal"):
            assert torch.equal(r[key].view(torch.int32) if key in ("depth", "normal") else r[key],
                               runs[0][key].view(torch.int32) if key in ("depth", "normal") else runs[0][key]), key


def _camera():
    wl = synth.workload("dmsr_study")
    c2w = np.eye(4, dtype=np.float32)
    c2w[:3] = np.asarray(wl["c2w"], dtype=np.float32)[:3]
    return wl, c2w


def test_grid_view_is_cast_grid_on_get_rays_k_and_batches_views(scene):
    wl, c2w = _camera()
    H, W = 48, 64
    K = np.asarray(wl["K"], dtype=np.float32).copy()
    K[0] *= W / wl["W"]
    K[1] *= H / wl["H"]
    poses = np.stack([c2w, synth.pose_spherical(30.0, -20.0, 4.0), synth.pose_spherical(-70.0, -35.0, 3.5)]).astype(np.float32)
    lut = np.random.default_rng(0).integers(0, 256, (scene["ins_num"] + 1, 3)).astype(np.uint8)
    args = (scene["occ"], scene["lab"], np.eye(4), H, W, K)
    batch = OB.grid_view(*args, torch.from_numpy(poses).to(DEV), wl["near"], wl["far"], EXT, scene["level"], lut=lut,
                         model_fine=scene["nf"])
    assert batch["depth"].shape == (3, H, W) and batch["image"].shape == (3, H, W, 3)
    assert batch["hit"].any()
    for v in range(3):
        one = OB.grid_view(*args, torch.from_numpy(poses[v]).to(DEV), wl["near"], wl["far"], EXT, scene["level"], lut=lut,
                           model_fine=scene["nf"])
        for key in ("depth", "label", "normal", "hit", "image"):
            assert torch.equal(batch[key][v], one[key]), (v, key)
        # the network may take another kernel for another number of points: the colours agree to its rounding
        assert torch.allclose(batch["rgb"][v], one["rgb"], atol=1e-5, rtol=0)
        o, d = get_rays_k(H, W, K, torch.from_numpy(poses[v]).to(DEV))
        c = OB.cast_grid(scene["occ"], scene["lab"], np.eye(4), o, d, wl["near"], wl["far"], EXT, scene["level"])
        for key in ("depth", "label", "normal", "hit"):
            assert torch.equal(one[key], c[key]), (v, key)
        # the network's colour at the hit points, the render's normalised direction
        dirs = d / torch.norm(d, dim=-1, keepdim=True)
        hit = c["hit"]
        with torch.no_grad():
            ref = torch.sigmoid(mlp_forward_points(scene["nf"], c["point"][hit], dirs[hit])[:, :3])
        assert torch.equal(one["rgb"][hit], ref)
        assert (one["rgb"][~hit] == 0).all() and (one["image"][~hit] == 0).all()


def test_piece_is_the_component_at_the_hit_voxel(scene):
    cc = OB.object_components(scene["occ"], scene["lab"], scene["level"])
    o, d, near, far = _frame_rays("dmsr_study")
    c = OB.cast_grid(scene["occ"], scene["lab"], np.eye(4), torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), near, far,
                     EXT, scene["level"], components=cc)
    hit = c["hit"]
    v = c["voxel"][hit]
    assert torch.equal(c["piece"][hit], cc["grid"][v[:, 0], v[:, 1], v[:, 2]])
    assert (c["piece"][~hit] == -1).all() and (c["piece"][hit] >= 0).all()
    # the point lies on the hit voxel's cube
    inv, b = E.grid_index_map(np.eye(4), EXT, scene["occ"].shape[0])
    u = (c["point"][hit].double().cpu().numpy() - b) @ inv.T
    assert (np.abs(u - v.cpu().numpy()) <= 0.5 + 1e-4).all()


def test_rejections_name_the_entry_point_and_write_nothing(scene):
    dim = scene["occ"].shape[0]
    n = 64
    o = torch.zeros((n, 3), device=DEV)
    d = torch.ones((n, 3), device=DEV)
    t = torch.full((n,), 7.0, device=DEV)
    lab = torch.full((n,), 7, dtype=torch.int16, device=DEV)
    vox = torch.full((n,), 7, dtype=torch.int32, device=DEV)
    nrm = torch.full((n, 3), 7.0, device=DEV)
    ctx = get_context(DEV)
    good = dict(occ=_lib.ptr(scene["occ"]), labels=_lib.ptr(scene["lab"], torch.int16), dim=dim, level=0.45,
                T=_lib.doubles(np.eye(4), 16), ext=_lib.doubles(EXT, 3), keep=None, o=_lib.ptr(o), d=_lib.ptr(d), n=n, near=0.0,
                far=10.0)
    flipped = np.eye(4)
    flipped[2, 2] = -1.0
    bad = [dict(dim=1), dict(dim=1291), dict(level=float("nan")), dict(level=float("inf")), dict(near=float("nan")),
           dict(far=float("inf")), dict(near=5.0, far=4.0), dict(n=-1), dict(occ=None), dict(labels=None), dict(o=None), dict(d=None),
           dict(T=_lib.doubles(flipped, 16)), dict(ext=_lib.doubles((1.0, 0.0, 1.0), 3)), dict(T=None)]
    for change in bad:
        a = dict(good, **change)
        with pytest.raises(RuntimeError, match="grid_cast"):
            ctx.call("dmnerf_grid_cast", ctx.handle, a["occ"], a["labels"], a["dim"], a["level"], a["T"], a["ext"], a["keep"], a["o"],
                     a["d"], a["n"], a["near"], a["far"], _lib.ptr(t), _lib.ptr(lab, torch.int16), _lib.ptr(vox, torch.int32),
                     _lib.ptr(nrm))
    torch.cuda.synchronize()
    assert (t == 7).all() and (lab == 7).all() and (vox == 7).all() and (nrm == 7).all()
    a = good
    with pytest.raises(RuntimeError, match="grid_cast: ctx is NULL"):
        ctx.call("dmnerf_grid_cast", None, a["occ"], a["labels"], a["dim"], a["level"], a["T"], a["ext"], a["keep"], a["o"], a["d"],
                 a["n"], a["near"], a["far"], _lib.ptr(t), _lib.ptr(lab, torch.int16), _lib.ptr(vox, torch.int32), _lib.ptr(nrm))


def test_move_objects_pick_moves_the_piece_under_the_pixel(scene, tmp_path):
    nc, nf = scene["nc"], scene["nf"]
    ins_num = scene["ins_num"]
    ck = tmp_path / "ck.tar"
    torch.save({"network_coarse_state_dict": {k: v.cpu() for k, v in nc.state_dict().items()},
                "network_fine_state_dict": {k: v.cpu() for k, v in nf.state_dict().items()}}, str(ck))
    wl, c2w = _camera()
    H, W = 24, 32
    K = np.asarray(wl["K"], dtype=np.float64).copy()
    K[0] *= W / wl["W"]
    K[1] *= H / wl["H"]
    np.save(str(tmp_path / "pose.npy"), c2w)
    np.save(str(tmp_path / "T.npy"), np.eye(4))
    # the sweep the tool splits (every label but the last) and the pixel whose ray hits it nearest the image centre
    with torch.no_grad():
        occ, lab = OB.occupancy_objects(nf, np.eye(4), OB.object_mask(ins_num, keep=range(ins_num)), 64, EXT, wl["near"], wl["far"],
                                        NI, device=DEV)
    lv = scene["level"]
    cc = OB.object_components(occ, lab, lv, 26)
    pose = torch.from_numpy(c2w).to(DEV)
    o, d = get_rays_k(H, W, K, pose)
    c = OB.cast_grid(occ, lab, np.eye(4), o, d, wl["near"], wl["far"], EXT, lv, components=cc)
    hits = torch.nonzero(c["hit"]).cpu().numpy()
    assert len(hits)
    y, x = hits[np.argmin(np.abs(hits - [H / 2, W / 2]).sum(1))]
    o1, d1 = get_rays_at(H, W, K, pose, [int(y) * W + int(x)])
    c1 = OB.cast_grid(occ, lab, np.eye(4), o1, d1, wl["near"], wl["far"], EXT, lv, components=cc)
    assert int(c1["piece"][0]) == int(c["piece"][y, x])
    out = tmp_path / "out"
    cmd = [sys.executable, os.path.join(ROOT, "tools", "move_objects.py"), str(ck), "--pose", str(tmp_path / "pose.npy"), "--hwk",
           str(H), str(W), *map(str, K.reshape(-1)), "--transform", str(tmp_path / "T.npy"), "--extents", *map(str, EXT),
           "--grid-dim", "64", "--level", str(lv), "--near", str(wl["near"]), "--far", str(wl["far"]), "--pick", str(int(x)),
           str(int(y)), "--mode", "translation", "--distance", "0.25", "--dilate", "0", "--preview", "--render", "none",
           "--out", str(out)]
    p = subprocess.run(cmd, capture_output=True, text=True, cwd=str(tmp_path))
    assert p.returncode == 0, p.stderr[-3000:]
    rec = json.loads(p.stdout.strip().splitlines()[-1])
    assert rec["pick"]["piece"] == int(c["piece"][y, x]) and rec["piece"] == rec["pick"]["piece"]
    assert rec["pick"]["label"] == int(c["label"][y, x]) == rec["label"]
    assert rec["render"] == "none" and rec["evaluated"] is None
    assert {"preview.png", "preview_edited.png", "preview_rgb.png", "transform.json"} <= set(rec["files"])
    assert "rgb.png" not in rec["files"] and "instance.png" not in rec["files"]
    # a pixel whose ray hits nothing fails clearly
    miss = torch.nonzero(~c["hit"]).cpu().numpy()
    if len(miss):
        my, mx = miss[0]
        cmd[cmd.index("--pick") + 1:cmd.index("--pick") + 3] = [str(int(mx)), str(int(my))]
        p = subprocess.run(cmd, capture_output=True, text=True, cwd=str(tmp_path))
        assert p.returncode != 0 and "hits no solid voxel" in p.stderr
