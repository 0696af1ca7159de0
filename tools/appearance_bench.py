#!/usr/bin/env python
"""Cost of object appearance (DESIGN.md, "Object appearance"): one JSON line with the frame rate of a 640 x 480 frame through the
frame driver at dmsr_study (ins_num 13) and replica_room0_93 (ins_num 93), rendered with a keep-all label selection (the
selected kernel without an edit), with a tint on every label, and with that tint plus density 0.3 on half the labels; and the
GPU's name and power limit read in the same run.
        python tools/appearance_bench.py [--reps 3]

Rays/s: median of --reps frames per variant, the variants alternated frame by frame after one warm-up frame each.  The
appearance is set and cleared around every frame, as render_frame does.  Nothing is written to disk."""
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


def frames(name, reps, dev):
    wl = synth.workload(name)
    ins_num = wl["ins_num"]
    nc, nf, _, _ = make_models(101, 202, ins_num, dev)
    H, W = 480, 640
    everything = list(range(ins_num + 1))
    tinted = {k: OB.tint((0.9, 0.3, 0.2)) for k in everything}
    variants = {"keep_all": {"keep_objects": everything},
                "tint_all": {"appearance": OB.Appearance(ins_num, colour=tinted)},
                "tint_density_half": {"appearance": OB.Appearance(ins_num, colour=tinted,
                                                                  density={k: 0.3 for k in everything[::2]})}}
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
    return {"workload": name, "ins_num": ins_num, "rays_per_s": rate,
            "tint_all_vs_keep_all": rate["tint_all"] / rate["keep_all"],
            "tint_density_half_vs_keep_all": rate["tint_density_half"] / rate["keep_all"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "tools/appearance_bench.py needs a CUDA device; there is no CPU fallback"
    dev = torch.device("cuda", 0)
    runs = [frames(n, a.reps, dev) for n in ("dmsr_study", "replica_room0_93")]
    try:
        gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as exc:
        gpu = "nvidia-smi unavailable: %s" % exc
    print(json.dumps({"metric": "object appearance cost", "reps": a.reps, "frames": runs, "gpu": gpu,
                      "gpu_name": torch.cuda.get_device_name(dev),
                      "what": "640x480 frames through the frame driver (host maps), rays/s median of %d, variants alternated"
                              % a.reps}))


if __name__ == "__main__":
    main()
