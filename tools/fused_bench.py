"""The fused render kernel alone: one 640x480 frame of rays (64 + 128 samples, want_raw=False, want_coarse=False) per call,
as bench.py renders it, for the exact and the fp16 network at ins_num 13 (dmsr_study) and 93 (replica_room0_93).  The four
configurations alternate inside one call; each is timed with CUDA events over --frames frames after warm-up, and the median
frame gives the rate.  The card name and its power limit are printed beside the rates, as one JSON line.

    python tools/fused_bench.py [--frames 7] [--warmup 2]
"""
import argparse
import json

import numpy as np
import torch

from _harness import alternate, cuda_device, gpu_identity
from dmnerf_b200 import _lib, synth
from dmnerf_b200.render import render_rays
from dmnerf_b200.testing import make_models

IMPLS = {"exact": _lib.IMPL_UMMA, "fp16": _lib.IMPL_UMMA_F16}
WORKLOADS = ("dmsr_study", "replica_room0_93")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    dev = cuda_device("fused_bench.py")
    calls = {}
    for w in WORKLOADS:
        wl = synth.workload(w)
        nc, nf, _, _ = make_models(101, 202, wl["ins_num"], dev)
        ro, rd = torch.from_numpy(wl["rays_o"]).to(dev), torch.from_numpy(wl["rays_d"]).to(dev)
        z = (torch.linspace(0, 1, 64) * (wl["far"] - wl["near"]) + wl["near"]).to(dev)
        for p, impl in IMPLS.items():
            calls[(w, p)] = (ro.shape[0], lambda ro=ro, rd=rd, nc=nc, nf=nf, z=z, impl=impl: render_rays(
                ro, rd, nc, nf, z, want_raw=False, want_coarse=False, want_samples=False, impl=impl))
    with torch.no_grad():
        ms = alternate({k: call for k, (_, call) in calls.items()}, a.frames, warmup=a.warmup)
    name, _, card = gpu_identity(dev)
    res = {"gpu": card[0] if card else name, "power_limit_w": card[1].removesuffix(" W") if card else None, "frame": [480, 640],
           "configs": []}
    for (w, p), (n, _) in calls.items():
        med = float(np.median(ms[(w, p)]))
        res["configs"].append({"workload": w, "ins_num": synth.workload(w)["ins_num"], "precision": p,
                               "frame_ms": [round(v, 3) for v in ms[(w, p)]], "median_ms": round(med, 3),
                               "rays_per_s": round(n / (med / 1e3), 1)})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
