#!/usr/bin/env python
"""Render chosen objects of a trained DM-NeRF checkpoint: each one alone, or the scene without them.

    python tools/render_objects.py CHECKPOINT.tar --pose POSE.npy --hwk H W K (--keep L [L ...] | --remove L [L ...]) --out DIR
           [--near 4 --far 15 --N-samples 64 --N-importance 128]

CHECKPOINT holds `network_coarse_state_dict` and `network_fine_state_dict` (the original's checkpoints).  POSE.npy holds one
camera-to-world pose [4, 4] (or [3, 4]) or several [N, 4, 4].  K is the 3x3 intrinsics, as a .npy file or as 9 numbers.  Writes
DIR/{i:03d}.png (RGBA: alpha = accumulated opacity, so an isolated object is a cut-out) and DIR/instance_{i:03d}.png (the
arg-max label; label k gets colour k of a fixed seeded palette)."""
import argparse
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np   # noqa: E402


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("checkpoint")
    ap.add_argument("--pose", required=True)
    ap.add_argument("--hwk", nargs="+", required=True, metavar="H W K", help="height, width and K (.npy file or 9 numbers)")
    sel = ap.add_mutually_exclusive_group(required=True)
    sel.add_argument("--keep", type=int, nargs="+", metavar="L", help="render only these object labels")
    sel.add_argument("--remove", type=int, nargs="+", metavar="L", help="render the scene without these object labels")
    ap.add_argument("--out", required=True)
    ap.add_argument("--near", type=float, default=4.0)
    ap.add_argument("--far", type=float, default=15.0)
    ap.add_argument("--N-samples", type=int, default=64)
    ap.add_argument("--N-importance", type=int, default=128)
    ap.add_argument("--device", default="cuda")
    a = ap.parse_args(argv)
    if len(a.hwk) not in (3, 11):
        ap.error("--hwk takes H W and K as a .npy path or as 9 numbers")
    a.H, a.W = int(a.hwk[0]), int(a.hwk[1])
    a.K = (np.load(a.hwk[2]) if len(a.hwk) == 3 else np.array([float(v) for v in a.hwk[2:]])).astype(np.float32).reshape(3, 3)
    return a


def main(argv=None):
    a = parse(argv)
    import torch
    from dmnerf_b200.embedder import get_embedder
    from dmnerf_b200.objects import render_objects
    from dmnerf_b200.testing import model_from_weights
    ck = torch.load(a.checkpoint, map_location="cpu")
    nets = [model_from_weights({k: v.float().numpy() for k, v in ck[key].items()}, a.device)
            for key in ("network_coarse_state_dict", "network_fine_state_dict")]
    poses = np.load(a.pose).astype(np.float32)
    if poses.ndim == 2:
        poses = poses[None]
    pe, _ = get_embedder(10)
    ve, _ = get_embedder(4)
    args = types.SimpleNamespace(near=a.near, far=a.far, N_samples=a.N_samples, N_importance=a.N_importance)
    maps = render_objects(pe, ve, nets[0], nets[1], poses, (a.H, a.W, a.K), args, keep=a.keep, remove=a.remove, savedir=a.out)
    print(json.dumps({"frames": len(maps), "mean_acc": [float(m["acc"].mean()) for m in maps],
                      "files": sorted(os.listdir(a.out))}))


if __name__ == "__main__":
    main()
