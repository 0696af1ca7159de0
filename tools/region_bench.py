#!/usr/bin/env python
"""Cost of region selection (DESIGN.md, "Region selection"): one JSON line with the frame rate of a 640 x 480 frame through the
frame driver at dmsr_study (ins_num 13) and replica_room0_93 (ins_num 93), rendered unselected, with a keep-all label selection
(the selected kernel without a region) and with a floater-cleanup region (the selected kernel with the per-sample look-up); the
time to build a region from a mask (region_from_mask: pack + dilate 1, 26-connectivity) at each --grid-dims; and the GPU's
name and power limit read in the same run.
        python tools/region_bench.py [--reps 3] [--grid-dims 256 512] [--sweep-dim 256]

Rays/s: median of --reps frames per variant, the variants alternated frame by frame after one warm-up frame each.  The floater
region is the component_region of each object label's largest 26-connected piece on a --sweep-dim labelled sweep of the bench
networks, dilated by one voxel: they scatter many small pieces over each label, so it is a stress case of the look-up rather
than a picture of a trained scene.  Build times: CUDA events, median of --reps after one warm-up, on a random mask of density
0.3.  Nothing is written to disk."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dmnerf_b200 import objects as OB                         # noqa: E402
from dmnerf_b200 import synth                                 # noqa: E402
from dmnerf_b200.render import render_frame                   # noqa: E402
from dmnerf_b200.testing import make_models                   # noqa: E402


def floater_region(nf, ins_num, dim, dev):
    T = np.eye(4)
    T[:3, 3] = (0.1, -0.2, 0.3)
    with torch.no_grad():
        occ, labels = OB.occupancy_objects(nf, T, OB.object_mask(ins_num, keep=range(ins_num)), dim, device=dev)
        s = occ.flatten()[::17].float()
        level = 0.45 if float(occ.min()) < 0.45 < float(occ.max()) else float(s.kthvalue(int(0.98 * s.numel())).values)
        cc = OB.object_components(occ, labels, level, 26)
    del occ, labels
    best = OB.largest_components(cc["label"], cc["voxels"])
    reg = OB.component_region(cc, [best[k] for k in sorted(best) if k != ins_num], T, dilate=1)
    return reg, {"pieces": int(cc["voxels"].shape[0]), "labels_with_pieces": len(best), "level": level}


def frames(name, reps, sweep_dim, dev):
    wl = synth.workload(name)
    ins_num = wl["ins_num"]
    nc, nf, _, _ = make_models(101, 202, ins_num, dev)
    reg, info = floater_region(nf, ins_num, sweep_dim, dev)
    H, W = 480, 640
    everything = list(range(ins_num + 1))
    variants = {"unselected": {}, "keep_all": {"keep_objects": everything}, "floater_region": {"region": reg}}
    times = {k: [] for k in variants}
    with torch.no_grad():
        for r in range(reps + 1):
            for k, kw in variants.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                render_frame(H, W, wl["K"], wl["c2w"], wl["near"], wl["far"], nc, nf, device=dev, **kw)
                torch.cuda.synchronize()
                if r:
                    times[k].append(time.perf_counter() - t0)
    rate = {k: H * W / float(np.median(v)) for k, v in times.items()}
    return {"workload": name, "ins_num": ins_num, "rays_per_s": rate, "sweep_dim": sweep_dim, **info,
            "keep_all_vs_unselected": rate["keep_all"] / rate["unselected"],
            "region_vs_keep_all": rate["floater_region"] / rate["keep_all"]}


def build_times(dim, reps, dev):
    mask = torch.rand((dim,) * 3, device=dev) < 0.3
    ms = []
    for r in range(reps + 1):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        OB.region_from_mask(mask, np.eye(4), dilate=1, connectivity=26)
        b.record()
        torch.cuda.synchronize()
        if r:
            ms.append(a.elapsed_time(b))
    return {"grid_dim": dim, "pack_dilate1_ms": float(np.median(ms)), "bits_MB": (dim ** 3 + 31) // 32 * 4 / 1e6}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--grid-dims", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--sweep-dim", type=int, default=256)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "tools/region_bench.py needs a CUDA device; there is no CPU fallback"
    dev = torch.device("cuda", 0)
    runs = [frames(n, a.reps, a.sweep_dim, dev) for n in ("dmsr_study", "replica_room0_93")]
    builds = [build_times(d, a.reps, dev) for d in a.grid_dims]
    try:
        gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as exc:
        gpu = "nvidia-smi unavailable: %s" % exc
    print(json.dumps({"metric": "region selection cost", "reps": a.reps, "frames": runs, "build": builds, "gpu": gpu,
                      "gpu_name": torch.cuda.get_device_name(dev),
                      "what": "640x480 frames through the frame driver (host maps), rays/s median of %d, variants alternated; "
                              "region build = pack + dilate 1 (26), CUDA events" % a.reps}))


if __name__ == "__main__":
    main()
