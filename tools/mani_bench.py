"""Per-frame device times of the manipulation loops at 640x480, ins_num 13, N_test 4096 on synthetic networks: the edited
render of one frame (manipulate_frame) with 1 moved object (the manipulator_eval shape) and with 3 (a manipulator_demo shape),
and manipulator_eval's per-frame metric block (PSNR, SSIM, gt ranks, ins_eval and its one read-back).  Prints one JSON line.
Network samples per pixel for m targets: (m + 1) * (448 + 128 m) at N_samples 64, N_importance 128.

    python tools/mani_bench.py [--frames 2] [--warmup 1]
"""
import argparse
import contextlib
import io
import json
import types

import numpy as np
import torch

from _harness import cuda_device, event_ms, gpu_identity, stages_ms
from dmnerf_b200 import synth, tester as T
from dmnerf_b200.manipulator import manipulate_frame, rigid_rays
from dmnerf_b200.embedder import get_embedder
from dmnerf_b200.testing import make_models

H, W, INS_NUM = 480, 640, 13


def _move(k):
    a = 0.15 * (k + 1)
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, -s, 0, 0.2 * k], [s, c, 0, -0.1], [0, 0, 1, 0.05 * k], [0, 0, 0, 1]], np.float32)


def one(m, frames, warmup, nc, nf, pe, ve, K, pose, args):
    args.target_labels = [2 + 3 * k for k in range(m)]
    tars = [rigid_rays(H, W, K, _move(k), pose) for k in range(m)]
    to, td = torch.stack([t[0] for t in tars]), torch.stack([t[1] for t in tars])
    ms = []
    for f in range(warmup + frames):
        t, out = event_ms(lambda: manipulate_frame(H, W, K, pose, to, td, pe, ve, nc, nf, args))
        if f >= warmup:
            ms.append(t)
    per_px = (m + 1) * (448 + 128 * m)
    med = float(np.median(ms))
    return {"targets": m, "frame_ms": [round(v, 1) for v in ms], "frame_ms_median": round(med, 1),
            "samples_per_pixel": per_px, "network_gsamples_per_s": round(per_px * H * W / (med / 1e3) / 1e9, 3)}, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    dev = cuda_device("mani_bench.py")
    wl = synth.workload("dmsr_study")
    K = np.array(wl["K"], dtype=np.float32)
    pose = torch.from_numpy(np.asarray(wl["c2w"], dtype=np.float32)).to(dev)
    nc, nf, _, _ = make_models(1, 2, INS_NUM, dev)
    pe, ve = get_embedder(10)[0], get_embedder(4)[0]
    args = types.SimpleNamespace(N_test=4096, near=float(wl["near"]), far=float(wl["far"]), N_samples=64, N_importance=128,
                                 ins_num=INS_NUM)
    cases = []
    with torch.no_grad():
        for m in (1, 3):
            res, out = one(m, a.frames, a.warmup, nc, nf, pe, ve, K, pose, args)
            cases.append(res)
            if m == 1:
                rgb, ins = out[0].reshape(H, W, 3).contiguous(), out[1]
        # manipulator_eval's metric block on the 1-target frame, against Voronoi gt objects
        rng = np.random.default_rng(0)
        gt_img = torch.from_numpy(rng.uniform(size=(H, W, 3)).astype(np.float32)).to(dev)
        yy, xx = np.mgrid[0:H, 0:W]
        seeds = rng.uniform(0, 1, (INS_NUM, 2)) * [H, W]
        dist = (yy[None] - seeds[:, 0, None, None]) ** 2 + (xx[None] - seeds[:, 1, None, None]) ** 2
        region = dist.argmin(0).astype(np.int32)
        labels = torch.from_numpy(region).to(dev).reshape(-1).contiguous()
        valid_gt = torch.unique(torch.from_numpy(region))
        scratch = torch.empty(H * W, device=dev, dtype=torch.int32), torch.empty(1, device=dev, dtype=torch.int32)

        def metrics(f):
            with contextlib.redirect_stdout(io.StringIO()):
                T._frame_metrics("mani_bench", f, rgb, gt_img, ins[:, :INS_NUM].contiguous(), labels, valid_gt, INS_NUM, None, *scratch)
        metric_ms = []
        for f in range(2 + 5):
            (t,), _ = stages_ms(lambda: metrics(f))     # one pair of events, reused every frame
            if f >= 2:
                metric_ms.append(t)
    name, _, card = gpu_identity(dev)
    name, power = card or (name, "unknown")
    print(json.dumps({"bench": "mani_frame_640x480", "gpu": name, "power_limit": power, "ins_num": INS_NUM, "N_test": args.N_test,
                      "cases": cases, "metrics_ms": [round(v, 3) for v in metric_ms],
                      "metrics_ms_median": round(float(np.median(metric_ms)), 3)}))


if __name__ == "__main__":
    main()
