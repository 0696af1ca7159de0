"""GPU: the native manipulation loops (manipulate_frame, manipulator_eval, manipulator_demo) against the original loops' own
output in tests/golden/mani_eval.npz (oracle/make_golden_mani_eval.py): target rays, chunking, teacher-forced files, the
end-to-end edit with the original's uniforms, and the inputs test_dmsr.py passes."""
import json
import os
import types

import numpy as np
import pytest
import torch

from dmnerf_b200 import synth
from test_metrics_host import read_png

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def gold(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "mani_eval.npz")))


def _models(g):
    from dmnerf_b200.testing import model_from_weights
    ins_num = int(g["ins_num"])
    wc, wf = synth.make_weights(int(g["seed_c"]), ins_num), synth.make_weights(int(g["seed_f"]), ins_num)
    wc["ins_linear.weight"], wc["ins_linear.bias"] = g["ins_w_c"], g["ins_b_c"]
    wf["ins_linear.weight"], wf["ins_linear.bias"] = g["ins_w_f"], g["ins_b_f"]
    return model_from_weights(wc, DEV).eval(), model_from_weights(wf, DEV).eval(), wc, wf


def _embedders():
    from dmnerf_b200.embedder import get_embedder
    return get_embedder(10)[0], get_embedder(4)[0]


def _scene(g, tmp_path, monkeypatch):
    (tmp_path / "data").mkdir(exist_ok=True)
    (tmp_path / "data" / "color_dict.json").write_text(json.dumps({"dmsr": {"study": json.loads(str(g["color_dict"]))}}))
    monkeypatch.chdir(tmp_path)
    return int(g["H"]), int(g["W"]), g["K"]


def _args(g, **kw):
    return types.SimpleNamespace(datadir="./data/dmsr/study", device=torch.device(DEV), ins_num=int(g["ins_num"]),
                                 N_test=int(g["n_test"]), N_samples=int(g["n_samples"]), N_importance=int(g["n_importance"]),
                                 near=float(g["near"]), far=float(g["far"]), **kw)


def _trans_dicts(g):
    return {"transformations": [{"mode": "translation", "transformation": g["eval_trans"].tolist()}]}


def _teacher(monkeypatch, rgbs, inss):
    """Replaces manipulate_frame with the original's maps, frame by frame."""
    import dmnerf_b200.manipulator as M
    it = iter(range(len(rgbs)))

    def fake(H, W, K, ori_pose, tar_o, tar_d, *a, **k):
        f = next(it)
        cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
        return cu(rgbs[f]), cu(inss[f]), None, None
    monkeypatch.setattr(M, "manipulate_frame", fake)


def _uniform_rand(seed, rows, n_importance, usum):
    """torch.rand stand-in: successive rows of the original run's uniform table (a seeded CPU torch.Generator)."""
    u = torch.rand(rows, n_importance, generator=torch.Generator().manual_seed(int(seed)))
    assert float(u.double().sum()) == float(usum)
    state = {"pos": 0}

    def rand(*size, **kw):
        shape = list(size[0]) if len(size) == 1 and isinstance(size[0], (list, tuple, torch.Size)) else list(size)
        n = int(np.prod(shape[:-1]))
        out = u[state["pos"]:state["pos"] + n].reshape(shape)
        state["pos"] += n
        return out.to(kw.get("device") or "cpu")
    return rand, state


def test_target_rays_match_the_original_arithmetic_bit_for_bit(gold):
    from dmnerf_b200.manipulator import rigid_rays, deformed_rays, deform_offsets
    from dmnerf_b200.helpers import get_rays_k
    g = gold
    H, W, K = int(g["H"]), int(g["W"]), g["K"]
    objs = json.loads(str(g["demo_deform_objs"]))
    objs_trans = json.loads(str(g["demo_objs_trans"]))
    for v, pose_np in enumerate(g["poses"]):
        pose = torch.from_numpy(pose_np).to(DEV)
        for name, tr in objs_trans.items():
            o, d = rigid_rays(H, W, K, tr[v]["transformation"], pose)
            ro, rd = get_rays_k(H, W, K, torch.tensor(tr[v]["transformation"], dtype=torch.float32, device=DEV) @ pose)
            assert torch.equal(o, ro.reshape(-1, 3)) and torch.equal(d, rd.reshape(-1, 3)), name
        ori_o, ori_d = (r.reshape(-1, 3) for r in get_rays_k(H, W, K, pose))
        for j, obj in enumerate(objs):
            off = deform_offsets(obj["deform_func"], H, v)
            o, d = deformed_rays(ori_o, ori_d, off, H, W)
            want = ori_o.cpu().numpy().copy()                                 # fp32 + fp64 -> fp64 sum, one rounding to fp32
            want[:, 0] = (want[:, 0].astype(np.float64) + np.repeat(g["demo_deform_offsets"][v, j], W)).astype(np.float32)
            assert np.array_equal(o.cpu().numpy(), want), obj["deform_func"]
            assert torch.equal(d, ori_d) and d.data_ptr() != ori_d.data_ptr()


def test_manipulate_frame_equals_manipulator_chunk_by_chunk(gold):
    """Preallocated outputs, a partial last chunk (768 = 300 + 300 + 168), and the default generator consumed as the loop of
    manipulator.py:246-269 consumes it."""
    from dmnerf_b200.manipulator import manipulate_frame, manipulator, rigid_rays
    from dmnerf_b200.helpers import get_rays_k
    g = gold
    nc, nf, _, _ = _models(g)
    pe, ve = _embedders()
    H, W, K = int(g["H"]), int(g["W"]), g["K"]
    args = _args(g, target_labels=[2, 7])
    pose = torch.from_numpy(g["poses"][1]).to(DEV)
    tars = [rigid_rays(H, W, K, t["transformation"], pose) for t in
            (json.loads(str(g["demo_objs_trans"]))["chair"][1], json.loads(str(g["demo_objs_trans"]))["lamp"][0])]
    to, td = torch.stack([t[0] for t in tars]), torch.stack([t[1] for t in tars])
    torch.cuda.manual_seed(7)
    got = manipulate_frame(H, W, K, pose, to, td, pe, ve, nc, nf, args)
    torch.cuda.manual_seed(7)
    o, d = (r.reshape(-1, 3) for r in get_rays_k(H, W, K, pose))
    parts = []
    for s in range(0, H * W, args.N_test):
        e = min(s + args.N_test, H * W)
        parts.append(manipulator(pe, ve, nc, nf, torch.stack([o[s:e], d[s:e]]), torch.stack([to[:, s:e], td[:, s:e]], 1), args))
    assert len(parts) == 3 and parts[-1][0].shape[0] == 168
    for k, what in enumerate(("rgb", "ins", "tar_rgb", "tar_ins_accum")):
        assert torch.equal(got[k], torch.cat([p[k] for p in parts])), what
    assert got[1].shape == (H * W, int(g["ins_num"]) + 1)


def _check_eval_files(g, out, H, W):
    d = out / "translation"
    for i in range(2):
        assert np.array_equal(read_png(d / f"{i}_rgb.png"), g["img_eval_%d_rgb" % i])
        assert np.array_equal(read_png(d / f"{i}_rgb_gt.png"), g["img_eval_%d_rgb_gt" % i])
        assert np.array_equal(read_png(d / f"{i}_ins.png"), g["img_eval_%d_ins" % i][..., ::-1])        # cv2 stores BGR
        assert np.array_equal(read_png(d / f"{i}_ins_gt.png"), g["img_eval_%d_ins_gt" % i][..., ::-1])
    assert json.loads((d / "matching_log.json").read_text()) == json.loads(str(g["eval_matching_log"]))
    got = np.loadtxt(d / "test_results.txt")
    want = np.loadtxt(str(g["eval_test_results"]).splitlines())
    assert got.shape == want.shape == (3, 9)
    np.testing.assert_allclose(got, want, rtol=0, atol=1.5e-6, equal_nan=True)
    assert np.isnan(got[:, 2]).all()


def test_teacher_forced_eval_writes_the_original_files(gold, tmp_path, monkeypatch, capsys):
    from dmnerf_b200.manipulator import manipulator_eval
    g = gold
    H, W, K = _scene(g, tmp_path, monkeypatch)
    nc, nf, _, _ = _models(g)
    _teacher(monkeypatch, g["eval_rgb"], g["eval_ins"])
    args = _args(g, target_label=int(g["eval_target_label"]))
    manipulator_eval(*_embedders(), nc, nf, g["poses"], (H, W, K), _trans_dicts(g), str(tmp_path / "out"), g["ins_rgbs"], args,
                     gt_rgbs=torch.from_numpy(g["eval_gt_rgbs"]), gt_labels=torch.from_numpy(g["eval_gt_labels"]))
    assert args.target_labels == [int(g["eval_target_label"])]
    _check_eval_files(g, tmp_path / "out", H, W)
    printed = capsys.readouterr().out
    assert printed.count("=" * 50) == 4 and "APs: [" in printed and "AP50: " in printed


@pytest.mark.parametrize("case", ["rigid", "deform"])
def test_teacher_forced_demo_writes_the_original_files(gold, tmp_path, monkeypatch, capsys, case):
    from dmnerf_b200.manipulator import manipulator_demo
    g = gold
    H, W, K = _scene(g, tmp_path, monkeypatch)
    nc, nf, _, _ = _models(g)
    _teacher(monkeypatch, g["demo_%s_rgb" % case], g["demo_%s_ins" % case])
    objs = json.loads(str(g["demo_%s_objs" % case]))
    args = _args(g, mani_type=case)
    manipulator_demo(*_embedders(), nc, nf, g["poses"], (H, W, K), json.loads(str(g["demo_objs_trans"])), str(tmp_path),
                     g["ins_rgbs"], objs, torch.from_numpy(g["poses"]), json.loads(str(g["demo_ins_map"])), args)
    assert args.target_labels == [o["tar_id"] for o in objs]
    for i in range(2):
        pre = "img_demo_%s_%d_" % (case, i)
        assert np.array_equal(read_png(tmp_path / case / f"{i}_rgb.png"), g[pre + "rgb"])
        assert np.array_equal(read_png(tmp_path / case / f"{i}_ins.png"), g[pre + "ins"][..., ::-1])
        assert np.array_equal(read_png(tmp_path / case / f"{i}_ins_pred_mask.png"), g[pre + "ins_pred_mask"])
    printed = capsys.readouterr().out
    assert "Image0: " in printed and "Image1: " in printed


def _agree(a, b, tol=2e-3):
    a = a.detach().cpu().double().numpy() if torch.is_tensor(a) else np.asarray(a, dtype=np.float64)
    b = b.detach().cpu().double().numpy() if torch.is_tensor(b) else np.asarray(b, dtype=np.float64)
    return float((np.abs(a - b).max(-1) <= tol).mean())


def test_eval_end_to_end_with_the_original_uniforms(gold, tmp_path, monkeypatch):
    """The real edit render, fed the uniforms the original drew.  The edit holds discrete decisions (arg-max labels, importance
    sampling), so the yardstick is the original's own arithmetic in fp64 on the same rays and uniforms: the native maps agree
    with the original's on at least as many pixels as that twin does, minus 0.05."""
    import dmnerf_b200.manipulator as M
    from oracle import dmnerf_oracle as O
    g = gold
    H, W, K = _scene(g, tmp_path, monkeypatch)
    nc, nf, wc, wf = _models(g)
    args = _args(g, target_label=int(g["eval_target_label"]))
    rows = 2 * 3 * H * W
    rand, state = _uniform_rand(g["eval_useed"], rows, args.N_importance, g["eval_usum"])
    real_frame, seen = M.manipulate_frame, []

    def recording(*a, **k):
        out = real_frame(*a, **k)
        seen.append((a[3], a[4], a[5], out))
        return out
    monkeypatch.setattr(M, "manipulate_frame", recording)
    monkeypatch.setattr(torch, "rand", rand)
    M.manipulator_eval(*_embedders(), nc, nf, g["poses"], (H, W, K), _trans_dicts(g), str(tmp_path / "out"), g["ins_rgbs"], args,
                       gt_rgbs=torch.from_numpy(g["eval_gt_rgbs"]), gt_labels=torch.from_numpy(g["eval_gt_labels"]))
    monkeypatch.undo()
    assert state["pos"] == rows
    u = torch.rand(rows, args.N_importance, generator=torch.Generator().manual_seed(int(g["eval_useed"]))).double()
    pos = 0
    from dmnerf_b200.helpers import get_rays_k
    for f, (pose, to, td, out) in enumerate(seen):
        o, d = (r.reshape(-1, 3).cpu().double() for r in get_rays_k(H, W, K, pose))
        to, td = to[0].cpu().double(), td[0].cpu().double()
        twin_rgb, twin_ins = [], []
        with torch.no_grad():
            for s in range(0, H * W, args.N_test):
                e = min(s + args.N_test, H * W)
                us = []
                for _ in range(3):
                    us.append(u[pos:pos + e - s])
                    pos += e - s
                r = O.manipulator(O.to_torch(wc, torch.float64), O.to_torch(wf, torch.float64), torch.stack([o[s:e], d[s:e]]),
                                  [torch.stack([to[s:e], td[s:e]])], args.N_samples, args.N_importance, args.near, args.far,
                                  [args.target_label], us=us)
                twin_rgb.append(r[0])
                twin_ins.append(r[1])
        for ours, tw, ref, what in ((out[0], torch.cat(twin_rgb), g["eval_rgb"][f], "rgb"),
                                    (out[1], torch.cat(twin_ins), g["eval_ins"][f], "ins")):
            r_ours, r_twin = _agree(ours, ref), _agree(tw, ref)
            print("mani_eval frame %d %s: ours %.3f, fp64 twin %.3f of pixels within 2e-3" % (f, what, r_ours, r_twin))
            assert r_ours >= r_twin - 0.05, (f, what, r_ours, r_twin)
    assert pos == rows


def _tree(d):
    return {str(p.relative_to(d)): p.read_bytes() for p in sorted(d.rglob("*")) if p.is_file()}


def test_eval_with_the_inputs_test_dmsr_passes_is_byte_identical(gold, tmp_path, monkeypatch):
    """test_dmsr.py: CUDA poses, CUDA gt images and int8 CUDA labels inside no_grad; the same files as numpy / CPU inputs, and
    two runs give the same bytes."""
    from dmnerf_b200.manipulator import manipulator_eval
    g = gold
    H, W, K = _scene(g, tmp_path, monkeypatch)
    nc, nf, _, _ = _models(g)
    pe, ve = _embedders()
    args = _args(g, target_label=int(g["eval_target_label"]))
    torch.manual_seed(3)
    manipulator_eval(pe, ve, nc, nf, g["poses"], (H, W, K), _trans_dicts(g), str(tmp_path / "a"), g["ins_rgbs"], args,
                     gt_rgbs=g["eval_gt_rgbs"], gt_labels=g["eval_gt_labels"].astype(np.int64))
    with torch.no_grad():
        torch.manual_seed(3)
        manipulator_eval(pe, ve, nc, nf, torch.from_numpy(g["poses"]).to(DEV), (H, W, K), _trans_dicts(g), str(tmp_path / "b"),
                         g["ins_rgbs"], args, gt_rgbs=torch.from_numpy(g["eval_gt_rgbs"]).to(DEV),
                         gt_labels=torch.from_numpy(g["eval_gt_labels"]).to(torch.int8).to(DEV))
    torch.manual_seed(3)
    manipulator_eval(pe, ve, nc, nf, g["poses"], (H, W, K), _trans_dicts(g), str(tmp_path / "c"), g["ins_rgbs"], args,
                     gt_rgbs=g["eval_gt_rgbs"], gt_labels=g["eval_gt_labels"].astype(np.int64))
    a, b, c = _tree(tmp_path / "a"), _tree(tmp_path / "b"), _tree(tmp_path / "c")
    assert len(a) == 4 * 2 + 2 and a == b == c


def test_eval_without_gt_writes_only_the_rgb_images(gold, tmp_path, monkeypatch):
    from dmnerf_b200.manipulator import manipulator_eval
    g = gold
    H, W, K = _scene(g, tmp_path, monkeypatch)
    nc, nf, _, _ = _models(g)
    _teacher(monkeypatch, g["eval_rgb"], g["eval_ins"])
    manipulator_eval(*_embedders(), nc, nf, g["poses"], (H, W, K), _trans_dicts(g), str(tmp_path / "out"), g["ins_rgbs"],
                     _args(g, target_label=2))
    d = tmp_path / "out" / "translation"
    assert sorted(p.name for p in d.iterdir()) == ["0_rgb.png", "1_rgb.png"]
    assert np.array_equal(read_png(d / "0_rgb.png"), g["img_eval_0_rgb"])


def test_eval_rejects_labels_outside_the_rank_range(gold, tmp_path, monkeypatch):
    from dmnerf_b200.manipulator import manipulator_eval
    g = gold
    H, W, K = _scene(g, tmp_path, monkeypatch)
    nc, nf, _, _ = _models(g)
    _teacher(monkeypatch, g["eval_rgb"], g["eval_ins"])
    lab = g["eval_gt_labels"].copy()
    lab[0, 0, 0] = -3
    with pytest.raises(ValueError, match="gt labels"):
        manipulator_eval(*_embedders(), nc, nf, g["poses"], (H, W, K), _trans_dicts(g), str(tmp_path / "out"), g["ins_rgbs"],
                         _args(g, target_label=2), gt_rgbs=g["eval_gt_rgbs"], gt_labels=lab)


def test_frame_metrics_without_a_gt_object(gold):
    """The shared per-frame block on a frame with no gt object: all six APs 1.0, an empty map and no predicted label."""
    from dmnerf_b200 import tester as T
    g = gold
    H, W, n = int(g["H"]), int(g["W"]), int(g["H"]) * int(g["W"])
    rgb = torch.from_numpy(g["eval_rgb"][0]).to(DEV).reshape(H, W, 3)
    ins = torch.from_numpy(g["eval_ins"][0][:, :-1].copy()).to(DEV)
    labels = torch.zeros(n, device=DEV, dtype=torch.int32)
    scratch = torch.empty(n, device=DEV, dtype=torch.int32), torch.empty(1, device=DEV, dtype=torch.int32)
    p, s, lp, ap, ins_map, pred = T._frame_metrics("test", 0, rgb, rgb, ins, labels, torch.zeros(0, dtype=torch.int64), 13, None,
                                                   *scratch)
    assert ap == [1.0] * 6 and ins_map == {} and p == np.inf and np.isnan(lp)
    assert torch.equal(pred, torch.full((n,), -1, device=DEV, dtype=torch.int64))
