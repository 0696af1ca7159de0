"""CPU: the evaluation-metric checker (oracle/metrics.py) against the golden fixture made from the original ins_eval, PSNR / SSIM
identities, the PNG writer and the drop-in resolution of networks.tester."""
import os
import struct
import subprocess
import sys
import zlib

import numpy as np
import pytest

from oracle import metrics as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DROPIN = os.path.join(ROOT, "dm-nerf_b200", "dropin")


def load_ins_cases(golden_dir):
    """Yields (tag, pred [H,W,K] float32, gt labels [H,W], ins_num, crop, expected dict) from tests/golden/ins_eval.npz."""
    g = np.load(os.path.join(golden_dir, "ins_eval.npz"))
    for tag in g["tags"]:
        tag = str(tag)
        pred = (g["q_" + tag].astype(np.float32) / np.float32(g["Q"])).astype(np.float32)
        yield (tag, pred, g["gt_" + tag].astype(np.int64), int(g["ins_num_" + tag]), bool(g["crop_" + tag]),
               {k: g[k + "_" + tag] for k in ("pred_label", "ap", "return_labels", "valid_gt")})


def gt_ranks(gt, valid):
    rank = np.searchsorted(valid, gt)
    ok = (rank < len(valid)) & (valid[np.minimum(rank, len(valid) - 1)] == gt)
    return np.where(ok, rank, -1)


def test_oracle_ins_eval_reproduces_the_original(golden_dir):
    tags = []
    for tag, pred, gt, k, crop, exp in load_ins_cases(golden_dir):
        valid = exp["valid_gt"]
        o = M.ins_eval(pred.reshape(-1, k), gt_ranks(gt, valid).reshape(-1), len(valid), k, (gt >= k).reshape(-1) if crop else None)
        np.testing.assert_array_equal(o["pred_label"], exp["pred_label"].reshape(-1))
        np.testing.assert_array_equal(o["return_labels"], exp["return_labels"])
        np.testing.assert_allclose(o["ap"], exp["ap"], rtol=0, atol=1e-6)
        tags.append(tag)
    assert len(tags) == 5
    # the fixture covers gt objects matched to empty columns
    assert any((e["return_labels"] == -1).any() for *_, e in load_ins_cases(golden_dir))


def test_psnr_ssim_identities():
    rng = np.random.default_rng(0)
    x = rng.uniform(size=(20, 23, 3)).astype(np.float32)
    assert M.ssim(x, x) == pytest.approx(1.0, abs=1e-12)
    assert M.psnr(x, x) == np.inf
    a, b = np.full((9, 11, 3), 0.25, np.float32), np.full((9, 11, 3), 0.75, np.float32)
    C1 = 0.01 ** 2
    assert M.ssim(a, b) == pytest.approx((2 * 0.25 * 0.75 + C1) / (0.25 ** 2 + 0.75 ** 2 + C1), rel=1e-12)
    assert M.psnr(a, b) == pytest.approx(10 * np.log10(1 / 0.25), rel=1e-12)
    with pytest.raises(ValueError):
        M.ssim(x[:6], x[:6])


def test_ssim_hand_computed_8x8():
    """The 2x2 interior of an 8x8 frame, every 7x7 window averaged explicitly."""
    rng = np.random.default_rng(1)
    x = rng.uniform(size=(8, 8, 3)).astype(np.float32)
    y = np.clip(x + rng.normal(0, 0.1, size=x.shape), 0, 1).astype(np.float32)
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    chans = []
    for ch in range(3):
        s = []
        for r in (3, 4):
            for c in (3, 4):
                wx = x[r - 3:r + 4, c - 3:c + 4, ch].astype(np.float64)
                wy = y[r - 3:r + 4, c - 3:c + 4, ch].astype(np.float64)
                ux, uy = wx.mean(), wy.mean()
                vx, vy = wx.var(ddof=1), wy.var(ddof=1)
                vxy = ((wx - ux) * (wy - uy)).sum() / 48
                s.append(((2 * ux * uy + C1) * (2 * vxy + C2)) / ((ux * ux + uy * uy + C1) * (vx + vy + C2)))
        chans.append(np.mean(s))
    assert M.ssim(x, y) == pytest.approx(np.mean(chans), abs=1e-12)


def test_calculate_ap_orders_ties_stably():
    ious = np.array([0.9, 0.1, 0.9, 0.6], np.float32)
    conf = np.array([0.5, 0.5, 0.2, 0.5], np.float32)
    # stable order: 0, 1, 3, 2 -> TP at 0.5: 1, 0, 1, 1
    ap = M.calculate_ap(ious, 4, conf)
    prec = np.array([1, 1 / 2, 2 / 3, 3 / 4], np.float32)
    assert ap[0] == pytest.approx(float(0.25 * 1 + 0.25 * prec[3] + 0.25 * prec[3]), abs=1e-7)


def _decode_png(path):
    """Minimal decoder of non-interlaced 8-bit grey / RGB PNGs (all five scanline filters)."""
    data = open(path, "rb").read()
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, idat, w = 8, b"", None
    while pos < len(data):
        ln, = struct.unpack(">I", data[pos:pos + 4])
        tag, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + ln]
        assert struct.unpack(">I", data[pos + 8 + ln:pos + 12 + ln])[0] == zlib.crc32(tag + body) & 0xffffffff
        if tag == b"IHDR":
            w, h, depth, ctype, _, _, interlace = struct.unpack(">IIBBBBB", body)
            assert depth == 8 and ctype in (0, 2) and interlace == 0
            nc = 3 if ctype == 2 else 1
        elif tag == b"IDAT":
            idat += body
        pos += 12 + ln
    raw = zlib.decompress(idat)
    stride = w * nc
    out = np.zeros((h, stride), np.int32)
    for r in range(h):
        f, line = raw[r * (stride + 1)], np.frombuffer(raw, np.uint8, stride, r * (stride + 1) + 1).astype(np.int32)
        prev = out[r - 1] if r else np.zeros(stride, np.int32)
        cur = np.zeros(stride, np.int32)
        for i in range(stride):
            a = cur[i - nc] if i >= nc else 0
            b, c = prev[i], (prev[i - nc] if i >= nc else 0)
            pred = [0, a, b, (a + b) // 2, None][f]
            if f == 4:
                p = a + b - c
                pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
                pred = a if pa <= pb and pa <= pc else (b if pb <= pc else c)
            cur[i] = (line[i] + pred) & 255
        out[r] = cur
    return out.astype(np.uint8).reshape(h, w, nc) if nc == 3 else out.astype(np.uint8)


def read_png(path):
    try:
        from PIL import Image
    except ImportError:
        return _decode_png(path)
    return np.asarray(Image.open(path))


def test_png_writer_round_trips(tmp_path):
    from dmnerf_b200.tester import write_png
    rng = np.random.default_rng(2)
    rgb = rng.integers(0, 256, (13, 17, 3), dtype=np.uint8)
    grey = rng.integers(0, 256, (9, 5), dtype=np.uint8)
    write_png(tmp_path / "rgb.png", rgb)
    write_png(tmp_path / "grey.png", grey)
    for decode in (read_png, _decode_png):
        np.testing.assert_array_equal(decode(tmp_path / "rgb.png"), rgb)
        np.testing.assert_array_equal(decode(tmp_path / "grey.png"), grey)
    with pytest.raises(ValueError):
        write_png(tmp_path / "bad.png", rgb.astype(np.float32))


def test_label_luts_follow_the_visualizer_rules():
    from dmnerf_b200.tester import gt_label_lut, pred_label_lut
    rgbs = np.array([[10, 20, 30], [40, 50, 60], [70, 80, 90], [1, 2, 3]])
    color_dict = {"0": 3, "2": 1, "5": 0}
    lut = gt_label_lut(rgbs, color_dict, 6)
    np.testing.assert_array_equal(lut[[0, 1, 2, 5]], [[1, 2, 3], [0, 0, 0], [40, 50, 60], [10, 20, 30]])
    lut = pred_label_lut({"4": 2, "1": 5}, rgbs, color_dict, 6)
    np.testing.assert_array_equal(lut[[1, 4, 0]], [[10, 20, 30], [40, 50, 60], [0, 0, 0]])
    with pytest.raises(KeyError):                                # a matched gt label without a colour: as the original
        pred_label_lut({"3": 7}, rgbs, color_dict, 6)


def test_lpips_falls_back_to_nan_when_the_model_cannot_be_built(monkeypatch):
    """lpips.LPIPS(net='vgg') fetches the VGG16 backbone through torchvision; when that fails (no cache, no network) the column
    is NaN with one warning instead of an exception.  A missing package behaves the same way."""
    import types
    from dmnerf_b200 import tester as T

    def offline(*a, **k):
        raise OSError("no network: cannot download vgg16 weights")

    monkeypatch.setitem(sys.modules, "lpips", types.SimpleNamespace(LPIPS=offline))
    monkeypatch.setattr(T, "_lpips_warned", False)
    with pytest.warns(UserWarning, match="could not be built.*no network"):
        assert T._lpips_model("cpu") is None
    monkeypatch.setitem(sys.modules, "lpips", None)                       # import lpips -> ImportError
    monkeypatch.setattr(T, "_lpips_warned", False)
    with pytest.warns(UserWarning, match="not installed"):
        assert T._lpips_model("cpu") is None


def _run(code, env_extra, cwd):
    env = {k: v for k, v in os.environ.items() if k not in ("DMNERF_REFERENCE_ROOT", "DMNERF_TESTER")}
    env.update(env_extra)
    env["PYTHONPATH"] = os.pathsep.join([DROPIN, ROOT])
    return subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=str(cwd))


def test_dropin_tester_resolution(tmp_path):
    """networks.tester serves the native render_test (no lpips / skimage / cv2 / imageio import); with no checkout,
    networks.evaluator serves the native ins_eval / calculate_ap; DMNERF_TESTER=reference loads the checkout's module."""
    code = r"""
import sys
import dmnerf_b200.tester as nt, dmnerf_b200.render as nr, dmnerf_b200.helpers as nh
from networks.tester import render_test
import networks.tester as T, networks.evaluator as E
assert render_test is nt.render_test and T.dm_nerf is nr.dm_nerf and T.get_rays_k is nh.get_rays_k
assert E.ins_eval is nt.ins_eval and E.calculate_ap is nt.calculate_ap
assert not {"lpips", "skimage", "cv2", "imageio"} & set(sys.modules)
print("ok")
"""
    r = _run(code, {}, tmp_path)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-3000:]
    (tmp_path / "ref" / "networks").mkdir(parents=True)
    (tmp_path / "ref" / "networks" / "tester.py").write_text(
        "from networks.render import dm_nerf\ndef render_test(*a, **k): return 'original'\n")
    code = r"""
import dmnerf_b200.render as nr
import networks.tester as T
assert T.render_test() == "original" and T.dm_nerf is nr.dm_nerf
print("ok")
"""
    r = _run(code, {"DMNERF_REFERENCE_ROOT": str(tmp_path / "ref"), "DMNERF_TESTER": "reference"}, tmp_path)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-3000:]
    r = _run("import networks.tester", {"DMNERF_TESTER": "reference"}, tmp_path)
    assert r.returncode != 0 and "DMNERF_REFERENCE_ROOT" in r.stderr
