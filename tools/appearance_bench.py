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

import numpy as np
import torch

from _harness import alternate, cuda_device, gpu_identity, host_ms
from dmnerf_b200 import objects as OB
from dmnerf_b200 import synth
from dmnerf_b200.render import render_frame
from dmnerf_b200.testing import make_models


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

    def frame(kw):
        return lambda: render_frame(H, W, wl["K"], wl["c2w"], wl["near"], wl["far"], nc, nf, device=dev, **kw)
    with torch.no_grad():
        ms = alternate({k: frame(kw) for k, kw in variants.items()}, reps, clock=host_ms)
    rate = {k: H * W / (float(np.median(v)) * 1e-3) for k, v in ms.items()}
    return {"workload": name, "ins_num": ins_num, "rays_per_s": rate,
            "tint_all_vs_keep_all": rate["tint_all"] / rate["keep_all"],
            "tint_density_half_vs_keep_all": rate["tint_density_half"] / rate["keep_all"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    dev = cuda_device("appearance_bench.py")
    runs = [frames(n, a.reps, dev) for n in ("dmsr_study", "replica_room0_93")]
    name, smi, _ = gpu_identity(dev)
    print(json.dumps({"metric": "object appearance cost", "reps": a.reps, "frames": runs, "gpu": smi, "gpu_name": name,
                      "what": "640x480 frames through the frame driver (host maps), rays/s median of %d, variants alternated"
                              % a.reps}))


if __name__ == "__main__":
    main()
