"""Per-frame device times of render_test at 640x480: the fused render of the frame and the device metrics (PSNR, SSIM, gt ranks
and ins_eval with its one result read-back), for ins_num 13 and 93, on synthetic networks.  Prints one JSON line.

    python tools/eval_bench.py [--frames 5] [--warmup 2]
"""
import argparse
import json
import types

import numpy as np
import torch

from _harness import cuda_device, gpu_identity, stages_ms
from dmnerf_b200 import synth, tester as T, _lib
from dmnerf_b200.engine import get_context
from dmnerf_b200.embedder import get_embedder
from dmnerf_b200.testing import make_models


def one(ins_num, frames, warmup, dev, H=480, W=640):
    wl = synth.workload("dmsr_study")
    K = np.array(wl["K"], dtype=np.float32).copy()
    K[0, 2], K[1, 2] = W / 2, H / 2
    c2w = np.asarray(wl["c2w"], dtype=np.float32)
    nc, nf, _, _ = make_models(1, 2, ins_num, dev)
    pe, ve = get_embedder(10)[0], get_embedder(4)[0]
    args = types.SimpleNamespace(N_test=H * W, near=float(wl["near"]), far=float(wl["far"]), N_samples=64, N_importance=128,
                                 perturb=0.0, is_train=False, N_ins=None)
    rng = np.random.default_rng(0)
    gt_img = torch.from_numpy(rng.uniform(size=(H, W, 3)).astype(np.float32)).to(dev)
    yy, xx = np.mgrid[0:H, 0:W]
    n_obj = min(ins_num, 80)
    seeds = rng.uniform(0, 1, (n_obj, 2)) * [H, W]
    region = np.zeros((H, W), np.int64)
    best = np.full((H, W), np.inf)
    for o in range(n_obj):                                       # Voronoi gt objects
        d = (yy - seeds[o, 0]) ** 2 + (xx - seeds[o, 1]) ** 2
        region = np.where(d < best, o, region)
        best = np.minimum(best, d)
    labels = torch.from_numpy(region.astype(np.int32)).to(dev).reshape(-1).contiguous()
    gt_num = int(np.unique(region).size)
    ctx = get_context(dev)
    gt_row = torch.empty(H * W, device=dev, dtype=torch.int32)
    n_valid = torch.empty(1, device=dev, dtype=torch.int32)

    def metrics(frame):
        rgb, ins = frame
        res = T._result_buffer(dev)
        T._image_into(rgb.reshape(H, W, 3), gt_img, res)
        ctx.call("dmnerf_ins_label_rows", _lib.ptr(labels, torch.int32), H * W, 128, _lib.ptr(gt_row, torch.int32),
                 _lib.ptr(n_valid, torch.int32))
        T._ins_eval_rows(ins, gt_row, gt_num, res)
        return T._read_result(res)
    render_ms, metric_ms = [], []
    with torch.no_grad():
        for f in range(warmup + frames):
            # the metrics are issued while the render runs: one event between them, one synchronise after both
            (t_render, t_metrics), (_, r) = stages_ms(lambda: T._render_frame_device(H, W, K, c2w, pe, ve, nc, nf, args, dev),
                                                      metrics)
            T._check_status(r)
            if f >= warmup:
                render_ms.append(t_render)
                metric_ms.append(t_metrics)
    return {"ins_num": ins_num, "gt_objects": gt_num, "render_ms": [round(v, 3) for v in render_ms],
            "metrics_ms": [round(v, 3) for v in metric_ms], "metrics_ms_median": round(float(np.median(metric_ms)), 3),
            "render_ms_median": round(float(np.median(render_ms)), 3), "psnr": r.psnr, "ssim": r.ssim, "ap50": r.ap[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    dev = cuda_device("eval_bench.py")
    name, _, card = gpu_identity(dev)
    name, power = card or (name, "unknown")
    out = {"bench": "eval_frame_640x480", "gpu": name, "power_limit": power,
           "cases": [one(k, a.frames, a.warmup, dev) for k in (13, 93)]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
