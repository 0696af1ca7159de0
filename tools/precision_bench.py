"""Exact network against the fp16 preview network (IMPL_UMMA_F16) on full 640x480 frames of dmsr_study (ins_num 13) and
replica_room0_93 (ins_num 93), synthetic trained-like networks, through the same frame entry point (render_frame: one fused
kernel per part of the frame, maps copied back to the host).  The two precisions alternate inside one call and are timed with
CUDA events after warm-up; fp16's rgb PSNR and arg-max label agreement are taken against the exact render of the same frame.
One manipulate_frame with one moved object is timed in both precisions too.  --profile adds the per-stage split
(dmnerf_profile_*) of the stage-by-stage path on 64 Ki rays for both.  Prints one JSON line, with the card and power limit.

    python tools/precision_bench.py [--reps 5] [--warmup 2] [--profile]
"""
import argparse
import ctypes as C
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from dmnerf_b200 import _lib, synth                        # noqa: E402
from dmnerf_b200.engine import get_context                 # noqa: E402
from dmnerf_b200.render import render_frame, render_rays   # noqa: E402
from dmnerf_b200.testing import make_models                # noqa: E402
from eval_bench import gpu_info                            # noqa: E402

IMPLS = {"exact": _lib.IMPL_UMMA, "fp16": _lib.IMPL_UMMA_F16}
STAGES = ("prep_z", "coarse_net", "coarse_composite", "hier_sample", "fine_net", "fine_composite")


def _timed(fn):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    out = fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]), out


def _psnr(a, b):
    mse = float(((a.double() - b.double()) ** 2).mean())
    return 10.0 * np.log10(1.0 / max(mse, 1e-300))


def frames(name, reps, warmup):
    wl = synth.workload(name)
    H, W = wl["H"], wl["W"]
    nc, nf, _, _ = make_models(101, 202, wl["ins_num"], "cuda")
    call = lambda impl: render_frame(H, W, wl["K"], wl["c2w"], wl["near"], wl["far"], nc, nf, impl=impl)
    ms = {k: [] for k in IMPLS}
    maps = {}
    with torch.no_grad():
        for r in range(warmup + reps):
            for k, impl in IMPLS.items():
                t, maps[k] = _timed(lambda: call(impl))
                if r >= warmup:
                    ms[k].append(t)
    med = {k: float(np.median(v)) for k, v in ms.items()}
    rate = {k: H * W / (med[k] / 1e3) for k in IMPLS}
    agree = float((maps["fp16"]["ins"].argmax(-1) == maps["exact"]["ins"].argmax(-1)).double().mean())
    return {"workload": name, "ins_num": wl["ins_num"], "frame": [H, W],
            "frame_ms": {k: [round(v, 2) for v in ms[k]] for k in IMPLS},
            "rays_per_s": {k: round(rate[k], 1) for k in IMPLS}, "speedup": round(rate["fp16"] / rate["exact"], 3),
            "rgb_psnr_db": round(_psnr(maps["fp16"]["rgb"], maps["exact"]["rgb"]), 2), "label_agreement": round(agree, 5),
            "finite": bool(torch.isfinite(maps["fp16"]["rgb"]).all())}


def manipulation(reps, warmup):
    from dmnerf_b200.embedder import get_embedder
    from dmnerf_b200.manipulator import manipulate_frame, rigid_rays
    wl = synth.workload("dmsr_study")
    H, W = wl["H"], wl["W"]
    nc, nf, _, _ = make_models(101, 202, wl["ins_num"], "cuda")
    pose = torch.from_numpy(wl["c2w"]).cuda()
    move = np.eye(4, dtype=np.float32)
    move[:3, 3] = (0.3, -0.2, 0.1)
    to, td = rigid_rays(H, W, wl["K"], move, pose)
    args = types.SimpleNamespace(N_test=4096, N_samples=64, N_importance=128, near=wl["near"], far=wl["far"], target_labels=[3],
                                 ins_num=wl["ins_num"])
    pe, ve = get_embedder(10)[0], get_embedder(4)[0]
    ms = {k: [] for k in IMPLS}
    rgb = {}
    for r in range(warmup + reps):
        for k, impl in IMPLS.items():
            torch.cuda.manual_seed(7)
            t, out = _timed(lambda: manipulate_frame(H, W, wl["K"], pose, to[None], td[None], pe, ve, nc, nf, args, impl=impl))
            rgb[k] = out[0]
            if r >= warmup:
                ms[k].append(t)
    med = {k: float(np.median(v)) for k, v in ms.items()}
    return {"targets": 1, "frame_ms": {k: [round(v, 1) for v in ms[k]] for k in IMPLS},
            "speedup": round(med["exact"] / med["fp16"], 3), "rgb_psnr_db": round(_psnr(rgb["fp16"], rgb["exact"]), 2)}


def stage_split(name, n=65536):
    """Per-stage device times (ms) of the stage-by-stage path (want_raw=True) for both precisions."""
    wl = synth.workload(name)
    nc, nf, _, _ = make_models(101, 202, wl["ins_num"], "cuda")
    ro, rd = torch.from_numpy(wl["rays_o"][:n]).cuda(), torch.from_numpy(wl["rays_d"][:n]).cuda()
    z = (torch.linspace(0, 1, 64) * (wl["far"] - wl["near"]) + wl["near"]).cuda()
    ctx = get_context("cuda")
    res = {}
    with torch.no_grad():
        for k, impl in IMPLS.items():
            render_rays(ro, rd, nc, nf, z, want_raw=True, impl=impl)
            _lib.check(ctx.lib.dmnerf_profile_enable(ctx.handle, 1), "dmnerf_profile_enable")
            render_rays(ro, rd, nc, nf, z, want_raw=True, impl=impl)
            buf = (C.c_float * 16)()
            _lib.check(ctx.lib.dmnerf_profile_read(ctx.handle, buf, 16), "dmnerf_profile_read")
            _lib.check(ctx.lib.dmnerf_profile_enable(ctx.handle, 0), "dmnerf_profile_enable")
            res[k] = {s: round(buf[i], 3) for i, s in enumerate(STAGES)}
    return {"workload": name, "rays": n, "stage_ms": res}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("precision_bench: needs a CUDA device")
    name, power = gpu_info()
    res = {"gpu": name, "power_limit": power, "frames": [frames(w, a.reps, a.warmup) for w in ("dmsr_study", "replica_room0_93")],
           "manipulate_frame": manipulation(max(1, a.reps // 2), 1)}
    if a.profile:
        res["stages"] = [stage_split(w) for w in ("dmsr_study", "replica_room0_93")]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
