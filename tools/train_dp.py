"""Data-parallel training step (dmnerf_b200.distributed.train_iteration) on the synthetic dmsr_study scene: penalizer on,
full-image selection, one rank per GPU over NCCL.  Prints one JSON line: world size, global rays N, ms per iteration (CUDA
events over the timed loop), device-busy ms per iteration (sum of kernel times from torch.profiler, in a separate pass), the
gradient all-reduce's time and share of the iteration (CUDA events around it) -- each the max over ranks -- and rays/s.

    python -m torch.distributed.run --nproc_per_node W tools/train_dp.py [--rays 3072] [--ins-num 13|93] [--steps 20] [--warmup 5]

Training on the original's data.  With DMNERF_REFERENCE_ROOT pointing at a checkout of the original (its datasets/ and config.py
importable), the loop of train_dmsr.py becomes, on every rank (not covered by the test suite):

    np.random.seed(0); torch.manual_seed(3)                       # the same seeds on every rank: the same draws
    for i in range(N_iters):
        img_i = np.random.choice(i_train)
        batch = get_select_full(images[img_i].to(dev), poses[img_i, :3, :4].to(dev), K, gt_labels[img_i].to(dev),
                                args.N_train) + (None,)           # get_select_crop(...) for ScanNet: it returns N_ins
        res = train_iteration(i, batch, model_coarse, model_fine, optimizer, args, z_val_coarse, group)
        if rank == 0 and i % args.i_print == 0:
            print(i, float(res["total"]), replicas_identical(params, group))
        if rank == 0 and i % args.i_save == 0:
            torch.save({"iteration": i, "network_coarse_state_dict": model_coarse.state_dict(),
                        "network_fine_state_dict": model_fine.state_dict(),
                        "optimizer_state_dict": optimizer.state_dict()}, path)       # the original's checkpoint format
"""
import argparse
import json
import os
import sys
import types

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dmnerf_b200 import synth                                             # noqa: E402
from dmnerf_b200.distributed import train_iteration                       # noqa: E402
import dmnerf_b200.distributed as D                                       # noqa: E402
from dmnerf_b200.helpers import get_select_full, z_val_sample             # noqa: E402
from dmnerf_b200.testing import make_models                              # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=3072)
    ap.add_argument("--ins-num", type=int, default=13)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_dp.py needs CUDA devices")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = "cuda:%d" % local
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device(dev))
    wl = synth.workload("dmsr_study")
    H, W = wl["H"], wl["W"]
    mc, mf, _, _ = make_models(201, 202, a.ins_num, dev)
    mc.train(); mf.train()
    opt = torch.optim.Adam(list(mc.parameters()) + list(mf.parameters()), lr=5e-4, betas=(0.9, 0.999))
    args = types.SimpleNamespace(perturb=1.0, N_importance=128, ins_num=a.ins_num, penalize=True, tolerance=0.05, deta_w=0.05,
                                 lrate=5e-4, lrate_decay=500)
    gen = torch.Generator().manual_seed(1)
    gt_rgb = torch.rand(H, W, 3, generator=gen).to(dev)
    gt_lab = (torch.arange(H * W).reshape(H, W) * min(a.ins_num - 1, 12) // (H * W)).to(torch.int16).to(dev)
    pose = torch.from_numpy(wl["c2w"]).float().to(dev)
    zc = z_val_sample(a.rays, float(wl["near"]), float(wl["far"]), 64, device=dev)
    np.random.seed(0)
    torch.manual_seed(3)

    # the gradient all-reduce, timed with events on the stream around it
    ar = []
    real_all_reduce = D.all_reduce_grads

    def timed_all_reduce(params, group=None):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        real_all_reduce(params, group)
        e1.record()
        ar.append((e0, e1))
    D.all_reduce_grads = timed_all_reduce

    def step(i):
        batch = get_select_full(gt_rgb, pose, wl["K"], gt_lab, a.rays) + (None,)
        return train_iteration(i, batch, mc, mf, opt, args, zc)

    for i in range(a.warmup):
        step(i)
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    ar.clear()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(a.steps):
        res = step(a.warmup + i)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.steps
    ar_ms = sum(x.elapsed_time(y) for x, y in ar) / a.steps
    loss = float(res["total"].sum())
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(3):
            step(a.warmup + a.steps + i)
        torch.cuda.synchronize()
    busy = sum(ev.device_time for ev in prof.events() if str(ev.device_type).endswith("CUDA")) / 3.0 / 1e3
    stats = torch.tensor([ms, ar_ms, busy], device=dev, dtype=torch.float64)
    if world > 1:
        every = torch.empty(world, 3, device=dev, dtype=torch.float64)
        dist.all_gather_into_tensor(every, stats)
        stats = every.max(0).values
    if rank == 0:
        ms_max, ar_max, busy_max = stats.tolist()
        print(json.dumps({"world": world, "n": a.rays, "ins_num": a.ins_num, "ms_per_iter": round(ms_max, 3),
                          "device_busy_ms": round(busy_max, 3), "allreduce_ms": round(ar_max, 3),
                          "allreduce_share": round(ar_max / ms_max, 4), "rays_per_s": round(a.rays / (ms_max / 1e3)),
                          "loss": loss, "gpu": torch.cuda.get_device_name(local)}))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
