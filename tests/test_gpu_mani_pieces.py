"""GPU: moving pieces (DESIGN.md, "Moving pieces").  The exchanger with pieces and the vote kernel bit for bit against
oracle/pieces_oracle.py, the path without regions unchanged, the whole edit against the oracle edit in fp32 and fp64,
rejections, and tools/move_objects.py."""
import ctypes as C
import json
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from dmnerf_b200 import _lib, synth
from dmnerf_b200 import objects as OB
from dmnerf_b200.engine import get_context
from dmnerf_b200.manipulator import ExchangePieces, exchanger, manipulate_frame, piece_vote, rigid_rays
from dmnerf_b200.testing import make_models
from oracle import dmnerf_oracle as O
from oracle import pieces_oracle as P

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"


def _transform():
    T = np.eye(4)
    T[:3, 3] = (0.1, -0.2, 0.3)
    return T


_SWEEPS = {}


def _sweep_pieces(ins_num):
    """The 3 largest pieces (labels may repeat: a label moved twice is judged move by move) of a dim-256 labelled sweep of the
    bench networks -> (components, [(label, piece)])."""
    if ins_num not in _SWEEPS:
        _, nf, _, _ = make_models(101, 202, ins_num, DEV)
        with torch.no_grad():
            occ, lab = OB.occupancy_objects(nf, _transform(), OB.object_mask(ins_num, keep=range(ins_num)), 256, device=DEV)
            s = occ.flatten()[::17].float()
            level = 0.45 if float(occ.min()) < 0.45 < float(occ.max()) else float(s.kthvalue(int(0.98 * s.numel())).values)
            cc = OB.object_components(occ, lab, level, 26)
        del occ, lab
        top = np.argsort(-cc["voxels"], kind="stable")[:3]
        assert len(top) == 3
        _SWEEPS[ins_num] = (cc, [(int(cc["label"][c]), int(c)) for c in top])
    return _SWEEPS[ins_num]


def _regions(kind, ins_num, m, outside, g):
    """(move labels, regions, anchors) of m moves; with 3 moves the middle one has no region.  anchors: grid indices [k, 3] of
    the first move's piece (None for random bits)."""
    if kind == "random":
        dim = 32
        words = (dim ** 3 + 31) // 32
        bits = torch.randint(-2 ** 31, 2 ** 31 - 1, (words,), generator=g, dtype=torch.int64).to(torch.int32).to(DEV)
        labels = [5] if m == 1 else [2, 5, 7]
        reg = OB.Region(bits, dim, OB.voxel_map(_transform(), dim), outside=outside)
        regions = [reg] * m
        anchors = None
    else:
        cc, best = _sweep_pieces(ins_num)
        labels = [k for k, _ in best[:m]]
        regions = [OB.component_region(cc, [c], _transform(), dilate=1, outside=outside) for _, c in best[:m]]
        anchors = torch.nonzero(cc["grid"] == best[0][1]).cpu().double().numpy()
    if m == 3:
        regions[1] = None
    return labels, regions, anchors


def _inputs(ins_num, labels, n, s, n_sets, g, anchors=None):
    """Seeded raws (labels biased towards the moved ones), accumulated maps, rays from inside the default sweep grid (half of them
    from points of a piece, with short steps, when anchors are given), depths."""
    c = ins_num + 5
    A, b = OB.grid_affine(_transform(), 256)
    out = []
    for _ in range(n_sets):
        raw = torch.randn((n, s, c), generator=g) * 2
        pick = torch.randint(0, len(labels), (n, s), generator=g)
        hot = torch.rand((n, s), generator=g) < 0.6
        ch = torch.tensor(labels)[pick] + 4
        raw.scatter_add_(-1, ch[..., None], torch.where(hot, 6.0, 0.0)[..., None])
        acc = torch.rand((n, c - 4), generator=g)
        acc[torch.arange(n), torch.tensor(labels)[torch.randint(0, len(labels), (n,), generator=g)]] += \
            (torch.rand(n, generator=g) < 0.7).float()
        idx = torch.rand((n, 3), generator=g).double().numpy() * 255
        rd = torch.randn((n, 3), generator=g) * 0.4
        if anchors is not None:
            pick = torch.randint(0, anchors.shape[0], (n // 2,), generator=g).numpy()
            idx[:n // 2] = anchors[pick] + torch.rand((n // 2, 3), generator=g).double().numpy() - 0.5
            rd[:n // 2] *= 0.1
        ro = torch.from_numpy(idx @ A.T + b).float()
        z = torch.sort(torch.rand((n, s), generator=g) * 4.0, -1).values
        out.append((raw, acc, ro, rd, z))
    return out


@pytest.mark.parametrize("ins_num", [13, 93])
@pytest.mark.parametrize("m", [1, 3])
@pytest.mark.parametrize("kind", ["random", "component"])
@pytest.mark.parametrize("outside", ["keep", "drop"])
def test_exchanger_and_vote_equal_the_oracle_bit_for_bit(ins_num, m, kind, outside):
    g = torch.Generator().manual_seed(ins_num * 100 + m * 10 + (kind == "random") * 2 + (outside == "keep"))
    labels, regions, anchors = _regions(kind, ins_num, m, outside, g)
    oregs = [None if r is None else P.region_of(r, ins_num) for r in regions]
    n, s = 384, 40
    sets = _inputs(ins_num, labels, n, s, m + 1, g, anchors)
    cu = lambda t: t.to(DEV).contiguous()
    # the vote on a "fine pass" of the original rays (every move) and of each target (its own move)
    w = torch.rand((n, s), generator=g) * 0.08
    ori_raw, ori_acc, ro, rd, oz = sets[0]
    got = piece_vote(cu(ori_raw), cu(oz), cu(w), cu(ro), cu(rd), labels, regions).cpu().numpy()
    want = P.piece_vote(ori_raw, oz, w, ro, rd, labels, oregs)
    assert np.array_equal(got, want)
    assert 0 < want[0].mean() < 1, "the votes do not separate"          # both outcomes occur
    for i in range(m):
        _, _, tro, trd, tz = sets[i + 1]
        assert np.array_equal(piece_vote(cu(sets[i + 1][0]), cu(tz), cu(w), cu(tro), cu(trd), [labels[i]], [regions[i]]).cpu().numpy(),
                              P.piece_vote(sets[i + 1][0], tz, w, tro, trd, [labels[i]], [oregs[i]]))
    # the exchange, on random votes so that every branch of the rule is reached
    ori_votes = (torch.rand((m, n), generator=g) < 0.5).to(torch.uint8)
    tar_votes = [(torch.rand(n, generator=g) < 0.5).to(torch.uint8) for _ in range(m)]
    tars = [x[0] for x in sets[1:]]
    taccs = [x[1] for x in sets[1:]]
    for rest in ("keep", "drop"):
        drop = [rest == "drop"] * m
        opieces = {"regions": oregs, "rest_drop": drop, "ori_rays": (ro, rd), "ori_z": oz,
                   "tar_rays": [(x[2], x[3]) for x in sets[1:]], "tar_zs": [x[4] for x in sets[1:]],
                   "ori_votes": ori_votes.numpy(), "tar_votes": [v.numpy() for v in tar_votes]}
        ref = P.exchanger_pieces(ori_raw, tars, ori_acc, taccs, labels, opieces)
        pieces = ExchangePieces(regions, drop, (cu(ro), cu(rd)), cu(oz), [(cu(x[2]), cu(x[3])) for x in sets[1:]],
                                [cu(x[4]) for x in sets[1:]], cu(ori_votes), [cu(v) for v in tar_votes])
        out, _, lab, tlab = exchanger(cu(ori_raw), [cu(t) for t in tars], cu(ori_acc), [cu(a) for a in taccs], labels, pieces=pieces)
        assert torch.equal(out.cpu(), ref[0]), rest
        assert torch.equal(lab.cpu(), ref[2]) and torch.equal(tlab.cpu(), ref[3]), rest
        whole = O.exchanger(ori_raw, tars, ori_acc, taccs, labels)[0]
        assert not torch.equal(ref[0], whole), "the pieces change nothing here"


# ------------------------------------------------------------------------------------------ the edit on the mani_eval scene
@pytest.fixture(scope="module")
def gold(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "mani_eval.npz")))


def _scene(g):
    from dmnerf_b200.testing import model_from_weights
    ins_num = int(g["ins_num"])
    wc, wf = synth.make_weights(int(g["seed_c"]), ins_num), synth.make_weights(int(g["seed_f"]), ins_num)
    wc["ins_linear.weight"], wc["ins_linear.bias"] = g["ins_w_c"], g["ins_b_c"]
    wf["ins_linear.weight"], wf["ins_linear.bias"] = g["ins_w_f"], g["ins_b_f"]
    from dmnerf_b200.embedder import get_embedder
    H, W, K = int(g["H"]), int(g["W"]), g["K"]
    args = types.SimpleNamespace(N_test=int(g["n_test"]), N_samples=int(g["n_samples"]), N_importance=int(g["n_importance"]),
                                 near=float(g["near"]), far=float(g["far"]), target_labels=[int(g["eval_target_label"])])
    pose = torch.from_numpy(g["poses"][0]).to(DEV)
    to, td = rigid_rays(H, W, K, g["eval_trans"], pose)
    return dict(nc=model_from_weights(wc, DEV).eval(), nf=model_from_weights(wf, DEV).eval(), wc=wc, wf=wf, H=H, W=W, K=K,
                args=args, pose=pose, to=to[None], td=td[None], pe=get_embedder(10)[0], ve=get_embedder(4)[0])


def _frame(sc, seed=7, **kw):
    torch.cuda.manual_seed(seed)
    return manipulate_frame(sc["H"], sc["W"], sc["K"], sc["pose"], sc["to"], sc["td"], sc["pe"], sc["ve"], sc["nc"], sc["nf"],
                            sc["args"], **kw)


def _checker_region(sc, g, outside):
    """A 3-D checkerboard of 2-voxel cells on a dim-64 grid over the cameras' view, applying to the moved label: whatever the
    label covers is split between the piece and the rest."""
    T, ext = OB.region_transform(*OB.camera_region(g["poses"], (sc["H"], sc["W"], sc["K"]), sc["args"].far))
    i = torch.arange(64, device=DEV) // 2
    mask = ((i[:, None, None] + i[None, :, None] + i[None, None, :]) % 2) == 0
    return OB.region_from_mask(mask, T, ext, applies=sc["args"].target_labels, outside=outside)


def test_without_a_region_the_edit_is_unchanged(gold):
    sc = _scene(gold)
    before = _lib.launch_count()
    plain = _frame(sc)
    n_plain = _lib.launch_count() - before
    before = _lib.launch_count()
    none = _frame(sc, pieces=[None], rest="drop")
    assert _lib.launch_count() - before == n_plain                 # no vote launch, the exchanger without pieces
    ones = OB.region_from_mask(torch.ones((16,) * 3, dtype=torch.bool, device=DEV), np.eye(4), outside="keep")
    for rest in ("keep", "drop"):
        all_ones = _frame(sc, pieces=[ones], rest=rest)
        for k in range(4):
            assert torch.equal(none[k], plain[k]) and torch.equal(all_ones[k], plain[k]), (rest, k)


def _agree(a, b, tol=2e-3):
    a = a.detach().cpu().double().numpy() if torch.is_tensor(a) else np.asarray(a, dtype=np.float64)
    b = b.detach().cpu().double().numpy() if torch.is_tensor(b) else np.asarray(b, dtype=np.float64)
    return float((np.abs(a - b).max(-1) <= tol).mean())


@pytest.mark.parametrize("rest,outside", [("keep", "keep"), ("drop", "drop")])
def test_edit_with_a_piece_end_to_end_against_the_oracle(gold, monkeypatch, rest, outside):
    """The whole edit with a piece region, fed uniforms the test draws, against the oracle edit (pieces_oracle.manipulator) in
    fp32; the yardstick is the same oracle in fp64: ours agrees with the fp32 oracle on at least as many pixels as the fp64 twin,
    minus 0.05 (the measure of test_eval_end_to_end_with_the_original_uniforms)."""
    sc = _scene(gold)
    H, W, args = sc["H"], sc["W"], sc["args"]
    region = _checker_region(sc, gold, outside)
    rows = 3 * H * W
    u = torch.rand(rows, args.N_importance, generator=torch.Generator().manual_seed(11))
    pos = {"p": 0}

    def rand(*size, **kw):
        shape = list(size[0]) if len(size) == 1 and isinstance(size[0], (list, tuple, torch.Size)) else list(size)
        k = int(np.prod(shape[:-1]))
        out = u[pos["p"]:pos["p"] + k].reshape(shape)
        pos["p"] += k
        return out.to(kw.get("device") or "cpu")
    monkeypatch.setattr(torch, "rand", rand)
    ours = _frame(sc, pieces=[region], rest=rest)
    monkeypatch.undo()
    assert pos["p"] == rows
    from dmnerf_b200.helpers import get_rays_k
    o, d = (r.reshape(-1, 3).cpu() for r in get_rays_k(H, W, sc["K"], sc["pose"]))
    to, td = sc["to"][0].cpu(), sc["td"][0].cpu()
    oreg = [P.region_of(region, int(gold["ins_num"]))]
    res = {}
    with torch.no_grad():
        for tag, dt in (("fp32", torch.float32), ("fp64", torch.float64), ("whole", torch.float32)):
            rgb, ins, p = [], [], 0
            for s in range(0, H * W, args.N_test):
                e = min(s + args.N_test, H * W)
                us = [u[p + k * (e - s):p + (k + 1) * (e - s)].to(dt) for k in range(3)]
                p += 3 * (e - s)
                r = P.manipulator(O.to_torch(sc["wc"], dt), O.to_torch(sc["wf"], dt), torch.stack([o[s:e], d[s:e]]).to(dt),
                                  [torch.stack([to[s:e], td[s:e]]).to(dt)], args.N_samples, args.N_importance, args.near, args.far,
                                  args.target_labels, us=us, regions=None if tag == "whole" else oreg,
                                  rest_drop=[rest == "drop"])
                rgb.append(r[0])
                ins.append(r[1])
            res[tag] = (torch.cat(rgb), torch.cat(ins))
    assert _agree(res["fp32"][0], res["whole"][0], 1e-6) < 1.0, "the piece region changes nothing in this frame"
    for k, what in enumerate(("rgb", "ins")):
        r_ours, r_twin = _agree(ours[k], res["fp32"][k]), _agree(res["fp64"][k], res["fp32"][k])
        print("pieces %s/%s %s: ours %.3f, fp64 twin %.3f of pixels within 2e-3" % (rest, outside, what, r_ours, r_twin))
        assert r_ours >= r_twin - 0.05, (what, r_ours, r_twin)


# ------------------------------------------------------------------------------------------ rejections
def test_rejections(gold):
    sc = _scene(gold)
    mv = sc["args"].target_labels[0]
    other = OB.region_from_mask(torch.ones((8,) * 3, dtype=torch.bool, device=DEV), np.eye(4), applies=[mv + 1])
    ok = OB.region_from_mask(torch.ones((8,) * 3, dtype=torch.bool, device=DEV), np.eye(4), applies=[mv])
    with pytest.raises(ValueError, match="applies"):
        _frame(sc, pieces=[other])
    with pytest.raises(ValueError, match="entries"):
        _frame(sc, pieces=[ok, None])
    for bad in ("move", ["keep", "drop"], ["maybe"]):
        with pytest.raises(ValueError, match="rest"):
            _frame(sc, pieces=[ok], rest=bad)
    elsewhere = OB.Region(ok.bits, ok.dim, ok.voxel_map, ok.applies)
    elsewhere.bits = ok.bits.to("cuda:1") if torch.cuda.device_count() > 1 else ok.bits.cpu()
    with pytest.raises(ValueError, match="live on"):
        _frame(sc, pieces=[elsewhere])
    # the C entry points: a NULL vote array, a bad dim and a label outside `applies` fail before any launch
    n, s, c = 64, 8, 18
    raw = torch.randn((n, s, c), device=DEV)
    acc = torch.rand((n, c - 4), device=DEV)
    ro, rd = torch.randn((n, 3), device=DEV), torch.randn((n, 3), device=DEV)
    z = torch.rand((n, s), device=DEV)
    votes = torch.ones(n, dtype=torch.uint8, device=DEV)
    ctx = get_context(DEV)
    lab = torch.empty((n, s), dtype=torch.int64, device=DEV)

    def call(edit):
        p = ExchangePieces([ok], [False], (ro, rd), z, [(ro, rd)], [z], votes[None], [votes])
        d, keep = p.describe([mv], n, s, c - 5, raw.device)
        edit(d)
        before = _lib.launch_count()
        rc = ctx.lib.dmnerf_exchanger(_lib.ptr(raw), _lib.ptrs([raw]), _lib.ptr(acc), _lib.ptrs([acc]), (C.c_int * 1)(mv), 1, n, s,
                                      c, _lib.ptr(lab, torch.int64), _lib.ptr(lab, torch.int64), C.byref(d), ctx.stream())
        assert _lib.launch_count() == before + (rc == 0)                 # a rejected call launches nothing
        return rc
    assert call(lambda d: None) == 0
    for edit in (lambda d: setattr(d, "ori_vote", (C.c_void_p * 8)()), lambda d: setattr(d, "tar_vote", (C.c_void_p * 8)()),
                 lambda d: setattr(d.region[0], "dim", 1), lambda d: setattr(d.region[0], "dim", 1291),
                 lambda d: setattr(d.region[0], "applies", (C.c_uint32 * 4)()), lambda d: setattr(d, "ori_z", None),
                 lambda d: setattr(d, "tar_z", (C.c_void_p * 8)())):
        assert call(edit) != 0
        assert len(ctx.lib.dmnerf_last_error()) > 0
    with pytest.raises(RuntimeError, match="applies"):
        bad = _lib.RegionDesc()
        bad.bits, bad.dim = ok.bits.data_ptr(), ok.dim
        ctx.call("dmnerf_piece_vote", _lib.ptr(raw), _lib.ptr(z), _lib.ptr(z), _lib.ptr(ro), _lib.ptr(rd), n, s, c,
                 (C.c_int * 1)(mv), (_lib.RegionDesc * 1)(bad), 1, _lib.ptr(votes, torch.uint8))
    ctx.sync_check()


# ------------------------------------------------------------------------------------------ the tool
@pytest.mark.parametrize("flags", [["--move-label", "{label}", "--rest", "drop"], ["--move-piece", "{piece}"]])
def test_move_objects_tool_writes_its_files(tmp_path, flags):
    nc, nf, _, _ = make_models(7, 8, 13, "cpu")
    ck = str(tmp_path / "ck.tar")
    torch.save({"network_coarse_state_dict": nc.state_dict(), "network_fine_state_dict": nf.state_dict()}, ck)
    wl = synth.workload("dmsr_study")
    H, W = 24, 32
    K = synth.dmsr_intrinsics(H, W)
    np.save(str(tmp_path / "pose.npy"), wl["c2w"])
    np.savetxt(str(tmp_path / "T.txt"), _transform())
    # the piece to move: the largest piece of the sweep the tool runs
    with torch.no_grad():
        nf_dev = nf.to(DEV)
        occ, lab = OB.occupancy_objects(nf_dev, _transform(), OB.object_mask(13, keep=range(13)), 48, None, 4.0, 15.0, 32,
                                        device=DEV)
        cc = OB.object_components(occ, lab, 0.0, 26)
    piece = int(np.argmax(cc["voxels"]))
    label = int(cc["label"][piece])
    out = str(tmp_path / "out")
    args = [f.format(label=label, piece=piece) for f in flags]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "move_objects.py"), ck, "--pose", str(tmp_path / "pose.npy"),
                        "--hwk", str(H), str(W)] + [repr(float(v)) for v in K.reshape(-1)] + args +
                       ["--mode", "translation", "--transform", str(tmp_path / "T.txt"), "--grid-dim", "48", "--level", "0.0",
                        "--N-samples", "16", "--N-importance", "32", "--N-test", "300", "--out", out],
                       capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert sorted(os.listdir(out)) == ["instance.png", "rgb.png", "transform.json"] == res["files"]
    assert res["label"] == label and res["piece"] == piece
    rec = json.loads(open(os.path.join(out, "transform.json")).read())
    assert np.asarray(rec["transformations"][0]["transformation"]).shape == (4, 4) and len(rec["centre"]) == 3
