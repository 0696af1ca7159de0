"""The fused render kernel alone: one 640x480 frame of rays (64 + 128 samples, want_raw=False, want_coarse=False) per call,
as bench.py renders it, for the exact and the fp16 network at ins_num 13 (dmsr_study) and 93 (replica_room0_93).  The four
configurations alternate inside one call; each is timed with CUDA events over --frames frames after warm-up, and the median
frame gives the rate.  The card name, its power limit and the SM clock sampled during the timed frames are printed beside the
rates, as one JSON line.

    python tools/fused_bench.py [--frames 7] [--warmup 2]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dmnerf_b200 import _lib, synth                        # noqa: E402
from dmnerf_b200.render import render_rays                 # noqa: E402
from dmnerf_b200.testing import make_models                # noqa: E402

IMPLS = {"exact": _lib.IMPL_UMMA, "fp16": _lib.IMPL_UMMA_F16}
WORKLOADS = ("dmsr_study", "replica_room0_93")


def smi(fields):
    """One nvidia-smi query of the current card (read only), or None where the tool is missing."""
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=" + fields,
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=20)
        return [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fused_bench: needs a CUDA device")
    dev = torch.device("cuda")
    calls = {}
    for w in WORKLOADS:
        wl = synth.workload(w)
        nc, nf, _, _ = make_models(101, 202, wl["ins_num"], dev)
        ro, rd = torch.from_numpy(wl["rays_o"]).to(dev), torch.from_numpy(wl["rays_d"]).to(dev)
        z = (torch.linspace(0, 1, 64) * (wl["far"] - wl["near"]) + wl["near"]).to(dev)
        for p, impl in IMPLS.items():
            calls[(w, p)] = (ro.shape[0], lambda ro=ro, rd=rd, nc=nc, nf=nf, z=z, impl=impl: render_rays(
                ro, rd, nc, nf, z, want_raw=False, want_coarse=False, want_samples=False, impl=impl))
    ms = {k: [] for k in calls}
    clocks = []
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    with torch.no_grad():
        for r in range(a.warmup + a.frames):
            for k, (_, call) in calls.items():
                ev[0].record()
                call()
                ev[1].record()
                if r >= a.warmup and k[1] == "exact":
                    c = smi("clocks.sm")            # sampled while the frame runs
                    if c:
                        clocks.append(int(c[0]))
                torch.cuda.synchronize()
                if r >= a.warmup:
                    ms[k].append(ev[0].elapsed_time(ev[1]))
    info = smi("name,power.limit,clocks.max.sm")
    res = {"gpu": info[0] if info else torch.cuda.get_device_name(0), "power_limit_w": info[1] if info else None,
           "max_sm_clock_mhz": info[2] if info else None,
           "sm_clock_mhz_during": {"median": float(np.median(clocks)), "min": min(clocks), "max": max(clocks)} if clocks else None,
           "frame": [480, 640], "configs": []}
    for (w, p), (n, _) in calls.items():
        med = float(np.median(ms[(w, p)]))
        res["configs"].append({"workload": w, "ins_num": synth.workload(w)["ins_num"], "precision": p,
                               "frame_ms": [round(v, 3) for v in ms[(w, p)]], "median_ms": round(med, 3),
                               "rays_per_s": round(n / (med / 1e3), 1)})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
