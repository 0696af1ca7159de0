"""GPU: the device-side test-view metrics (csrc/metrics.cu) against the CPU checker (oracle/metrics.py) and the golden fixture made
from the original ins_eval, and render_test end to end through the drop-in import."""
import json
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import metrics as M
from test_metrics_host import load_ins_cases, gt_ranks, read_png

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def frames(H, W, seed):
    rng = np.random.default_rng(seed)
    yield "random", rng.uniform(size=(H, W, 3)).astype(np.float32), rng.uniform(size=(H, W, 3)).astype(np.float32)
    yy, xx = np.mgrid[0:H, 0:W] / max(H, W)
    smooth = np.stack([np.sin(3 * yy + 1), np.cos(2 * xx), np.sin(yy * xx * 5)], -1) * 0.5 + 0.5
    yield "smooth", smooth.astype(np.float32), np.clip(smooth + rng.normal(0, 0.02, smooth.shape), 0, 1).astype(np.float32)


@pytest.mark.parametrize("H,W", [(7, 7), (61, 83), (480, 640)])
def test_psnr_ssim_match_the_checker(H, W):
    from dmnerf_b200.tester import image_metrics
    for name, a, b in frames(H, W, H * W):
        p, s = image_metrics(torch.from_numpy(a).to(DEV), torch.from_numpy(b).to(DEV))
        assert p == pytest.approx(M.psnr(a, b), rel=1e-9), name
        assert abs(s - M.ssim(a, b)) <= 1e-8, (name, s, M.ssim(a, b))
    x = torch.from_numpy(a).to(DEV)
    p, s = image_metrics(x, x)
    assert p == np.inf and s == pytest.approx(1.0, abs=1e-12)


def test_small_frames_are_rejected():
    from dmnerf_b200.tester import ssim
    with pytest.raises(ValueError):
        ssim(torch.zeros(6, 9, 3, device=DEV), torch.zeros(6, 9, 3, device=DEV))
    with pytest.raises(RuntimeError):
        ssim(torch.zeros(8, 8, 3), torch.zeros(8, 8, 3))


def _dense_gt(gt, ins_num, crop):
    """tester.py:97-112: one-hot gt in the first valid columns."""
    gt_t = torch.from_numpy(gt)
    valid = torch.unique(gt_t)
    if crop:
        valid = valid[:-1]
    gt_ins = torch.zeros(gt.shape + (ins_num,))
    gt_ins[..., :len(valid)] = F.one_hot(gt_t.long())[..., valid.long()].float()
    return gt_ins, len(valid), valid.numpy()


def test_ins_eval_matches_the_original_on_the_golden_frames(golden_dir):
    from dmnerf_b200.tester import ins_eval
    for tag, pred, gt, k, crop, exp in load_ins_cases(golden_dir):
        gt_ins, gt_num, _ = _dense_gt(gt, k, crop)
        mask = torch.from_numpy((gt < k).astype(np.float32)).to(DEV) if crop else None
        pl, ap, ret = ins_eval(torch.from_numpy(pred).to(DEV), gt_ins.to(DEV), gt_num, k, mask)
        assert pl.shape == gt.shape and pl.dtype == torch.int64
        np.testing.assert_array_equal(pl.cpu().numpy(), exp["pred_label"], err_msg=tag)
        np.testing.assert_array_equal(ret, exp["return_labels"], err_msg=tag)
        np.testing.assert_allclose(ap, exp["ap"], rtol=0, atol=1e-6, err_msg=tag)


def synthetic_instance_frame(rng, H, W, ins_num, n_gt):
    ids = np.sort(rng.choice(ins_num, n_gt, replace=False))
    seeds = rng.uniform(0, 1, (n_gt, 2)) * [H, W]
    yy, xx = np.mgrid[0:H, 0:W]
    region = np.argmin((yy[..., None] - seeds[:, 0]) ** 2 + (xx[..., None] - seeds[:, 1]) ** 2, -1)
    hot = rng.permutation(ins_num)[:n_gt][region]
    hot = np.where(rng.uniform(size=(H, W)) < 0.1, rng.integers(0, ins_num, (H, W)), hot)
    logits = rng.normal(0, 1, (H, W, ins_num)).astype(np.float32)
    np.put_along_axis(logits, hot[..., None], np.take_along_axis(logits, hot[..., None], -1) + 4, -1)
    e = np.exp(logits - logits.max(-1, keepdims=True))
    return (e / e.sum(-1, keepdims=True)).astype(np.float32), ids[region]


def _native_vs_oracle(pred, gt, k, crop=False):
    from dmnerf_b200.tester import ins_eval
    gt_ins, gt_num, valid = _dense_gt(gt, k, crop)
    mask = torch.from_numpy((gt < k).astype(np.float32)).to(DEV) if crop else None
    pl, ap, ret = ins_eval(torch.from_numpy(pred).to(DEV), gt_ins.to(DEV), gt_num, k, mask)
    o = M.ins_eval(pred.reshape(-1, k), gt_ranks(gt, valid).reshape(-1), gt_num, k, (gt >= k).reshape(-1) if crop else None)
    np.testing.assert_array_equal(pl.cpu().numpy().reshape(-1), o["pred_label"])
    np.testing.assert_array_equal(ret, o["return_labels"])
    np.testing.assert_allclose(ap, o["ap"], rtol=0, atol=1e-6)
    return pl, ap, ret


def test_ins_eval_matches_the_checker_at_480x640_ins93():
    rng = np.random.default_rng(93)
    pred, gt = synthetic_instance_frame(rng, 480, 640, 93, 70)
    _native_vs_oracle(pred, gt, 93)


def test_confidence_ties_keep_gt_order():
    """Two matched labels with the same median confidence and IoUs on both sides of a threshold: the stable rule decides."""
    rng = np.random.default_rng(5)
    H, W, k = 40, 60, 13
    gt = np.zeros((H, W), np.int64)
    gt[:, 20:40], gt[:, 40:] = 1, 2
    lab = gt.copy()
    lab[:12, 20:40] = 5                                   # gt 1 keeps IoU 560/800 = 0.7: a TP at 0.5, an FP at 0.75
    pred = rng.uniform(0, 0.05, (H, W, k)).astype(np.float32)
    np.put_along_axis(pred, lab[..., None], np.float32(0.75), -1)
    pl, ap, ret = _native_vs_oracle(pred, gt, k)
    assert ret.tolist() == [0, 1, 2]


def test_results_are_deterministic():
    from dmnerf_b200.tester import ins_eval, image_metrics
    rng = np.random.default_rng(7)
    pred, gt = synthetic_instance_frame(rng, 240, 320, 59, 30)
    gt_ins, gt_num, _ = _dense_gt(gt, 59, False)
    p, g = torch.from_numpy(pred).to(DEV), gt_ins.to(DEV)
    a = ins_eval(p, g, gt_num, 59)
    b = ins_eval(p, g, gt_num, 59)
    assert torch.equal(a[0], b[0]) and a[1] == b[1] and np.array_equal(a[2], b[2])
    x, y = torch.rand(240, 320, 3, device=DEV), torch.rand(240, 320, 3, device=DEV)
    assert image_metrics(x, y) == image_metrics(x, y)


def test_ins_eval_rejects_nan_and_cpu_tensors():
    from dmnerf_b200.tester import ins_eval
    pred = torch.rand(8, 8, 13, device=DEV)
    gt = torch.zeros(8, 8, 13, device=DEV)
    gt[..., 0] = 1
    pred[3, 4, 2] = float("nan")
    with pytest.raises(RuntimeError, match="NaN"):
        ins_eval(pred, gt, 1, 13)
    with pytest.raises(RuntimeError):
        ins_eval(pred.cpu(), gt.cpu(), 1, 13)


def test_calculate_ap_wrapper_matches_the_checker():
    from dmnerf_b200.tester import calculate_ap
    rng = np.random.default_rng(3)
    ious = rng.uniform(size=37).astype(np.float32)
    conf = rng.uniform(size=37).astype(np.float32)
    np.testing.assert_allclose(calculate_ap(torch.from_numpy(ious).to(DEV), 40, torch.from_numpy(conf).to(DEV)),
                               M.calculate_ap(ious, 40, conf), rtol=0, atol=1e-6)
    np.testing.assert_allclose(calculate_ap(torch.from_numpy(ious).to(DEV), 37), M.calculate_ap(ious, 37), rtol=0, atol=1e-6)


# ----------------------------------------------------------------------------------------------------------------- render_test
def _scene(tmp_path, ins_num, H, W, n_frames, crop):
    from dmnerf_b200 import synth
    rng = np.random.default_rng(11 + crop)
    wl = synth.workload("dmsr_study")
    K = np.array(wl["K"], dtype=np.float32).copy()
    K[0, 2], K[1, 2] = W / 2, H / 2
    c2w = np.asarray(wl["c2w"], dtype=np.float32)
    poses = []
    for f in range(n_frames):
        p = c2w.copy()
        p[:3, 3] += np.float32(0.05 * f)
        poses.append(p)
    gt_imgs = torch.from_numpy(rng.uniform(size=(n_frames, H, W, 3)).astype(np.float32))
    yy, xx = np.mgrid[0:H, 0:W]
    labels = []
    for f in range(n_frames):
        lab = (yy * 3 // H) * 3 + (xx * 3 // W) + f            # 9 blocks, ids shifted per frame
        if crop:
            lab = np.where((yy + xx + f) % 7 == 0, 250, lab)   # ScanNet-style unlabelled id >= ins_num
        labels.append(lab)
    gt_labels = torch.from_numpy(np.stack(labels).astype(np.int64))
    ins_rgbs = rng.integers(0, 256, (260, 3))
    color_dict = {str(i): i for i in range(0, 20)}
    color_dict["250"] = 255
    (tmp_path / "data").mkdir()
    (tmp_path / "data" / "color_dict.json").write_text(json.dumps({"dmsr": {"study": color_dict}}))
    return K, poses, gt_imgs, gt_labels, ins_rgbs, color_dict


def _import_dropin_render_test():
    drop = os.path.join(ROOT, "dm-nerf_b200", "dropin")
    saved = {k: v for k, v in sys.modules.items() if k == "networks" or k.startswith("networks.")}
    for k in saved:
        del sys.modules[k]
    old_ref = os.environ.pop("DMNERF_REFERENCE_ROOT", None)
    sys.path.insert(0, drop)
    try:
        from networks.tester import render_test
    finally:
        sys.path.remove(drop)
        for k in [k for k in sys.modules if k == "networks" or k.startswith("networks.")]:
            del sys.modules[k]
        sys.modules.update(saved)
        if old_ref is not None:
            os.environ["DMNERF_REFERENCE_ROOT"] = old_ref
    return render_test


@pytest.mark.parametrize("crop", [False, True])
def test_render_test_end_to_end(tmp_path, monkeypatch, crop):
    from dmnerf_b200.testing import make_models
    from dmnerf_b200.embedder import get_embedder
    from dmnerf_b200.render import render_frame
    from dmnerf_b200 import tester as T
    render_test = _import_dropin_render_test()
    assert render_test is T.render_test
    ins_num, H, W, n_frames = 13, 24, 40, 3
    K, poses, gt_imgs, gt_labels, ins_rgbs, color_dict = _scene(tmp_path, ins_num, H, W, n_frames, crop)
    monkeypatch.chdir(tmp_path)
    nc, nf, _, _ = make_models(3, 4, ins_num, DEV)
    args = types.SimpleNamespace(datadir="./data/dmsr/study", ins_num=ins_num, N_test=300, near=4.0, far=15.0, N_samples=64,
                                 N_importance=128, perturb=0.0, is_train=False, N_ins=None, device=torch.device(DEV))
    crop_mask = None
    oh, ow = H, W
    if crop:
        cm = np.zeros((H, W), np.int64)
        cm[2:H - 2, 3:W - 3] = 1
        crop_mask = torch.from_numpy(cm)
        oh, ow = H - 4, W - 6
        args.crop_height, args.crop_width = oh, ow
    out = tmp_path / "out"
    out.mkdir()
    render_test(get_embedder(10)[0], get_embedder(4)[0], nc, nf, poses, (H, W, K), args, gt_imgs=gt_imgs, gt_labels=gt_labels,
                ins_rgbs=ins_rgbs, savedir=str(out), crop_mask=crop_mask)

    rows, log = [], {}
    sel = None if crop_mask is None else crop_mask.reshape(-1).numpy() == 1
    for i, c2w in enumerate(poses):
        # the maps render_test evaluates are render_frame's, bit for bit
        dev_rgb, dev_ins = T._render_frame_device(H, W, K, c2w, get_embedder(10)[0], get_embedder(4)[0], nc, nf, args,
                                                   torch.device(DEV))
        fr = render_frame(H, W, K, torch.from_numpy(c2w), 4.0, 15.0, nc, nf)
        assert torch.equal(dev_rgb.cpu(), fr["rgb"].reshape(-1, 3)) and torch.equal(dev_ins.cpu(), fr["ins"].reshape(-1, ins_num))
        rgb, ins = fr["rgb"].reshape(-1, 3).numpy(), fr["ins"].reshape(-1, ins_num).numpy()
        gt_img, gt_lab = gt_imgs[i].reshape(-1, 3).numpy(), gt_labels[i].reshape(-1).numpy()
        if sel is not None:
            rgb, ins, gt_img, gt_lab = rgb[sel], ins[sel], gt_img[sel], gt_lab[sel]
        rgb, gt_img, gt_lab = rgb.reshape(oh, ow, 3), gt_img.reshape(oh, ow, 3), gt_lab.reshape(oh, ow)
        valid = np.unique(gt_lab)
        if crop:
            valid = valid[:-1]
        o = M.ins_eval(ins, gt_ranks(gt_lab, valid).reshape(-1), len(valid), ins_num, (gt_lab >= ins_num).reshape(-1) if crop else None)
        rows.append([M.psnr(rgb, gt_img), M.ssim(rgb, gt_img), np.nan] + list(o["ap"]))
        ins_map = {str(l): int(valid[g]) for g, l in enumerate(o["return_labels"]) if l != -1}
        log[str(i)] = ins_map

        np.testing.assert_array_equal(read_png(out / ("%03d.png" % i)), (255 * np.clip(rgb, 0, 1)).astype(np.uint8))
        lut = T.pred_label_lut(ins_map, ins_rgbs, color_dict, ins_num + 1)
        np.testing.assert_array_equal(read_png(out / ("instance_%03d.png" % i)), lut[o["pred_label"]].reshape(oh, ow, 3)[..., ::-1])
        glut = T.gt_label_lut(ins_rgbs, color_dict, 251)
        np.testing.assert_array_equal(read_png(out / ("%d_ins_gt.png" % i)), glut[gt_lab][..., ::-1])
        np.testing.assert_array_equal(read_png(out / ("%d_ins_gt_mask.png" % i)), gt_lab.astype(np.uint8))
    rows = np.array(rows)
    expected = np.concatenate([rows, rows.mean(0, keepdims=True)], 0)          # the LPIPS column is NaN without lpips
    got = np.loadtxt(out / "test_results.txt")
    assert got.shape == (n_frames + 1, 9)
    np.testing.assert_allclose(got, expected, rtol=0, atol=2e-6, equal_nan=True)
    assert json.loads((out / "matching_log.json").read_text()) == log


def test_render_test_as_the_training_loop_calls_it(tmp_path, monkeypatch):
    """train_dmsr.py:97-103: poses as torch.Tensor(poses.to(device)) (CUDA), CPU float gt images, CUDA int16 gt labels, inside
    torch.no_grad() with args.is_train False.  Same files as a call with numpy poses and CPU labels."""
    from dmnerf_b200.testing import make_models
    from dmnerf_b200.embedder import get_embedder
    render_test = _import_dropin_render_test()
    ins_num, H, W, n_frames = 13, 20, 28, 2
    K, poses, gt_imgs, gt_labels, ins_rgbs, _ = _scene(tmp_path, ins_num, H, W, n_frames, False)
    monkeypatch.chdir(tmp_path)
    nc, nf, _, _ = make_models(7, 8, ins_num, DEV)
    args = types.SimpleNamespace(datadir="./data/dmsr/study", ins_num=ins_num, N_test=250, near=4.0, far=15.0, N_samples=64,
                                 N_importance=128, perturb=0.0, is_train=False, N_ins=None, device=torch.device(DEV))
    pe, ve = get_embedder(10)[0], get_embedder(4)[0]
    (tmp_path / "host").mkdir()
    (tmp_path / "dev").mkdir()
    render_test(pe, ve, nc, nf, poses, (H, W, K), args, gt_imgs=gt_imgs, gt_labels=gt_labels, ins_rgbs=ins_rgbs,
                savedir=str(tmp_path / "host"))
    with torch.no_grad():
        test_poses = torch.Tensor(torch.from_numpy(np.stack(poses)).to(args.device))
        assert test_poses.is_cuda
        render_test(pe, ve, nc, nf, test_poses, (H, W, K), args, gt_imgs=gt_imgs, gt_labels=gt_labels.to(torch.int16).to(args.device),
                    ins_rgbs=ins_rgbs, savedir=str(tmp_path / "dev"), matched_file=str(tmp_path / "dev" / "matching_log.txt"))
    names = sorted(p.name for p in (tmp_path / "host").iterdir())
    assert names == sorted(p.name for p in (tmp_path / "dev").iterdir()) and len(names) == 4 * n_frames + 2
    for name in names:
        assert (tmp_path / "host" / name).read_bytes() == (tmp_path / "dev" / name).read_bytes(), name


def test_render_test_without_gt_writes_only_images(tmp_path, monkeypatch):
    from dmnerf_b200.testing import make_models
    from dmnerf_b200.embedder import get_embedder
    from dmnerf_b200.tester import render_test
    K, poses, _, _, ins_rgbs, _ = _scene(tmp_path, 13, 16, 20, 2, False)
    monkeypatch.chdir(tmp_path)
    nc, nf, _, _ = make_models(5, 6, 13, DEV)
    args = types.SimpleNamespace(datadir="./data/dmsr/study", ins_num=13, N_test=1000, near=4.0, far=15.0, N_samples=64,
                                 N_importance=128, perturb=0.0, is_train=False, N_ins=None, device=torch.device(DEV))
    render_test(get_embedder(10)[0], get_embedder(4)[0], nc, nf, poses, (16, 20, K), args, ins_rgbs=ins_rgbs, savedir=str(tmp_path))
    assert sorted(p.name for p in tmp_path.glob("*.png")) == ["000.png", "001.png"]
