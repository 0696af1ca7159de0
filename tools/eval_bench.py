"""Per-frame device times of render_test at 640x480: the fused render of the frame and the device metrics (PSNR, SSIM, gt ranks
and ins_eval with its one result read-back), for ins_num 13 and 93, on synthetic networks.  Prints one JSON line.

    python tools/eval_bench.py [--frames 5] [--warmup 2]
"""
import argparse
import json
import os
import subprocess
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dmnerf_b200 import synth, tester as T, _lib          # noqa: E402
from dmnerf_b200.engine import get_context                 # noqa: E402
from dmnerf_b200.embedder import get_embedder              # noqa: E402
from dmnerf_b200.testing import make_models                # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=20).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def one(ins_num, frames, warmup, H=480, W=640):
    dev = torch.device("cuda")
    wl = synth.workload("dmsr_study")
    K = np.array(wl["K"], dtype=np.float32).copy()
    K[0, 2], K[1, 2] = W / 2, H / 2
    c2w = np.asarray(wl["c2w"], dtype=np.float32)
    nc, nf, _, _ = make_models(1, 2, ins_num, "cuda")
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
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    render_ms, metric_ms = [], []
    with torch.no_grad():
        for f in range(warmup + frames):
            ev[0].record()
            rgb, ins = T._render_frame_device(H, W, K, c2w, pe, ve, nc, nf, args, dev)
            ev[1].record()
            res = T._result_buffer(dev)
            T._image_into(rgb.reshape(H, W, 3), gt_img, res)
            ctx.call("dmnerf_ins_label_rows", _lib.ptr(labels, torch.int32), H * W, 128, _lib.ptr(gt_row, torch.int32),
                     _lib.ptr(n_valid, torch.int32))
            T._ins_eval_rows(ins, gt_row, gt_num, res)
            r = T._read_result(res)
            ev[2].record()
            torch.cuda.synchronize()
            T._check_status(r)
            if f >= warmup:
                render_ms.append(ev[0].elapsed_time(ev[1]))
                metric_ms.append(ev[1].elapsed_time(ev[2]))
    return {"ins_num": ins_num, "gt_objects": gt_num, "render_ms": [round(v, 3) for v in render_ms],
            "metrics_ms": [round(v, 3) for v in metric_ms], "metrics_ms_median": round(float(np.median(metric_ms)), 3),
            "render_ms_median": round(float(np.median(render_ms)), 3), "psnr": r.psnr, "ssim": r.ssim, "ap50": r.ap[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    name, power = gpu_info()
    out = {"bench": "eval_frame_640x480", "gpu": name, "power_limit": power,
           "cases": [one(k, a.frames, a.warmup) for k in (13, 93)]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
