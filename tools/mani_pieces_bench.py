#!/usr/bin/env python
"""Cost of moving pieces (DESIGN.md, "Moving pieces"): one JSON line with the device time of a 640 x 480 edited frame
(manipulate_frame, args.N_test rays per edit call, one moved label translated) at dmsr_study (ins_num 13) and replica_room0_93
(ins_num 93), edited three ways: the whole label (the reference's edit), one piece of it with rest="keep", and with rest="drop";
the device time of the two streaming kernels alone at one edit call's sizes; and the GPU's name and power limit.
        python tools/mani_pieces_bench.py [--reps 2] [--sweep-dim 256] [--n-test 4096]

Frames: CUDA events around each frame on the current stream, median of --reps after one warm-up frame each, the three variants
alternated frame by frame.  The piece is the largest 26-connected component of a --sweep-dim labelled sweep of the bench
networks (its label is the moved one), as a component_region dilated by one voxel.  Kernels: dmnerf_piece_vote on a fine pass
(N_test rays, 64 + 128 samples) and dmnerf_exchanger with and without the piece on the second exchange's sizes (64 + 128 + 128
samples), on random network outputs; median of 20 launches after 3 warm-ups.  Nothing is written to disk."""
import argparse
import json
import types

import numpy as np
import torch

from _harness import alternate, cuda_device, event_ms, gpu_identity
from dmnerf_b200 import objects as OB
from dmnerf_b200 import synth
from dmnerf_b200.embedder import get_embedder
from dmnerf_b200.manipulator import ExchangePieces, exchanger, manipulate_frame, piece_vote, rigid_rays
from dmnerf_b200.testing import make_models


def largest_piece(nf, ins_num, dim, dev):
    T = np.eye(4)
    T[:3, 3] = (0.1, -0.2, 0.3)
    with torch.no_grad():
        occ, labels = OB.occupancy_objects(nf, T, OB.object_mask(ins_num, keep=range(ins_num)), dim, device=dev)
        s = occ.flatten()[::17].float()
        level = 0.45 if float(occ.min()) < 0.45 < float(occ.max()) else float(s.kthvalue(int(0.98 * s.numel())).values)
        cc = OB.object_components(occ, labels, level, 26)
    del occ, labels
    piece = int(np.argmax(cc["voxels"]))
    label = int(cc["label"][piece])
    info = {"pieces_of_label": int((cc["label"] == label).sum()), "piece_voxels": int(cc["voxels"][piece]),
            "label_voxels": int(cc["voxels"][cc["label"] == label].sum()), "level": level}
    return OB.component_region(cc, [piece], T, dilate=1), label, info


def frames(name, reps, sweep_dim, n_test, dev):
    wl = synth.workload(name)
    ins_num = wl["ins_num"]
    nc, nf, _, _ = make_models(101, 202, ins_num, dev)
    region, label, info = largest_piece(nf, ins_num, sweep_dim, dev)
    H, W, K = wl["H"], wl["W"], wl["K"]
    pose = torch.as_tensor(wl["c2w"], dtype=torch.float32, device=dev)
    trans = OB.manipulation_transform(np.zeros(3), "translation")["transformations"][0]["transformation"]
    tar_o, tar_d = rigid_rays(H, W, K, trans, pose)
    args = types.SimpleNamespace(N_test=n_test, N_samples=64, N_importance=128, near=wl["near"], far=wl["far"],
                                 target_labels=[label])
    pe, ve = get_embedder(10)[0], get_embedder(4)[0]
    variants = {"whole_label": {}, "piece_keep": {"pieces": [region], "rest": "keep"},
                "piece_drop": {"pieces": [region], "rest": "drop"}}

    def frame(kw):
        return lambda: manipulate_frame(H, W, K, pose, tar_o[None], tar_d[None], pe, ve, nc, nf, args, **kw)
    with torch.no_grad():
        ms = alternate({k: frame(kw) for k, kw in variants.items()}, reps)
    frame_ms = {k: float(np.median(v)) for k, v in ms.items()}
    return {"workload": name, "ins_num": ins_num, "moved_label": label, "sweep_dim": sweep_dim, **info, "frame_ms": frame_ms,
            "piece_keep_vs_whole": frame_ms["piece_keep"] / frame_ms["whole_label"],
            "piece_drop_vs_whole": frame_ms["piece_drop"] / frame_ms["whole_label"],
            "kernels": kernels(wl, region, label, ins_num, n_test, dev)}


def kernels(wl, region, label, ins_num, n, dev):
    g = torch.Generator(device=dev).manual_seed(3)
    c = ins_num + 5
    ro = torch.as_tensor(wl["rays_o"][:n], device=dev).float().contiguous()
    rd = torch.as_tensor(wl["rays_d"][:n], device=dev).float().contiguous()

    def depths(s):
        return torch.sort(wl["near"] + (wl["far"] - wl["near"]) * torch.rand((n, s), generator=g, device=dev), -1).values

    def raw(s):
        return torch.randn((n, s, c), generator=g, device=dev) * 3
    s_fine, s_two = 64 + 128, 64 + 128 + 128
    raw_f, z_f = raw(s_fine), depths(s_fine)
    w_f = torch.rand((n, s_fine), generator=g, device=dev) * 0.02
    ori, tar, z_o, z_t = raw(s_two), raw(s_two), depths(s_two), depths(s_two)
    acc_o, acc_t = torch.rand((n, c - 4), generator=g, device=dev), torch.rand((n, c - 4), generator=g, device=dev)
    votes = piece_vote(raw_f, z_f, w_f, ro, rd, [label], [region])
    pieces = ExchangePieces([region], [False], (ro, rd), z_o, [(ro, rd)], [z_t], votes, [votes[0]])
    work = ori.clone()
    calls = {"piece_vote": lambda: piece_vote(raw_f, z_f, w_f, ro, rd, [label], [region]),
             "exchanger": lambda: exchanger(work, [tar], acc_o, [acc_t], [label]),
             "exchanger_pieces": lambda: exchanger(work, [tar], acc_o, [acc_t], [label], pieces=pieces)}
    out = {}
    for k, fn in calls.items():
        t = []
        for r in range(23):
            work.copy_(ori)
            x, _ = event_ms(fn)
            if r >= 3:
                t.append(x)
        out[k + "_ms"] = float(np.median(t))
    out.update({"rays": n, "vote_samples": s_fine, "exchange_samples": s_two, "channels": c})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--sweep-dim", type=int, default=256)
    ap.add_argument("--n-test", type=int, default=4096)
    a = ap.parse_args()
    dev = cuda_device("mani_pieces_bench.py")
    runs = [frames(n, a.reps, a.sweep_dim, a.n_test, dev) for n in ("dmsr_study", "replica_room0_93")]
    name, smi, _ = gpu_identity(dev)
    print(json.dumps({"metric": "moving pieces cost", "reps": a.reps, "runs": runs, "gpu": smi, "gpu_name": name,
                      "what": "640x480 edited frames (manipulate_frame, N_test %d), CUDA events, median of %d, variants "
                              "alternated; kernels: median of 20 launches" % (a.n_test, a.reps)}))


if __name__ == "__main__":
    main()
