#!/usr/bin/env python
"""Looking at the labelled grid without the network (DESIGN.md, "Viewing the labelled grid"): one JSON line with
  grid_view     one 640x480 camera of the seeded keep-all sweep ("dmsr_study", ins_num 13) at grid_dim 256 and 512: device ms per
                frame (CUDA events), M rays/s, and the cast kernel's own device time (torch.profiler, a run of its own after the
                timing);
  look          for one move of the sweep's largest label at grid_dim 256: edited_grid + grid_view (the preview of the edit)
                against render_moves + render_frame(moves=) (the network render of the same move), alternating in each round,
                host clock around a synchronised call;
  colour        for one and for three moves at grid_dim 256: edited_grid + grid_view(model_fine=, moves=, source=) (the preview in
                the edit's network colour) against render_moves + render_frame(moves=) of the same moves, alternating, host clock;
                and the preview's device stages apart (CUDA events): the cast, the replay (dmnerf_grid_edit_source) and the network
                query at the hit pixels;
and the GPU's name and power limit read in the same run.  Median of --reps rounds after --warmup.
    python tools/grid_view_bench.py [--reps 5] [--warmup 1]"""
import argparse
import json

import numpy as np
import torch

from _harness import alternate, cuda_device, event_ms, gpu_identity, host_ms, stages_ms
from dmnerf_b200 import objects as OB
from dmnerf_b200 import synth
from dmnerf_b200.autograd import mlp_forward_points
from dmnerf_b200.helpers import get_rays_k
from dmnerf_b200.render import render_frame
from dmnerf_b200.testing import make_models

EXT, S, NI, CHUNK = (8.0, 8.0, 8.0), 64, 128, 8192


def _med(v):
    return round(float(np.median(v)), 3)


def _kernel_ms(fn):
    """Device time of the cast kernel alone in one profiled call (the rest of grid_view is ray generation and copies)."""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return round(sum(e.device_time_total for e in prof.key_averages() if "grid_cast_kernel" in e.key) / 1e3, 3)


def _colour(occ, labels, T, H, W, K, pose, near, far, level, nc, nf, dev, n_moves, a):
    """The coloured preview of n_moves moves (the largest labels, each by 8 voxels along its own axis) against their network
    render, and the preview's device stages."""
    dim = occ.shape[0]
    k, c = torch.unique(labels[occ > level], return_counts=True)
    order = [int(v) for v in k[torch.argsort(c, descending=True, stable=True)]]
    A, _ = OB.grid_affine(T, dim, EXT)
    moves = []
    for label, delta in zip(order, ([8.0, 0.0, 0.0], [0.0, 0.0, 8.0], [-8.0, 0.0, 0.0])[:n_moves]):
        m = np.eye(4)
        m[:3, 3] = A @ np.asarray(delta)
        moves.append((label, m))
    source = (occ, labels)

    def preview():
        e_occ, e_labels, _ = OB.edited_grid(occ, labels, T, moves, EXT, level)
        moved = OB.render_moves(occ, labels, T, moves, EXT, level, near, far, NI)
        return OB.grid_view(e_occ, e_labels, T, H, W, K, pose, near, far, EXT, level, model_fine=nf, moves=moved, source=source)

    def render():
        moved = OB.render_moves(occ, labels, T, moves, EXT, level, near, far, NI)
        return render_frame(H, W, K, pose, near, far, nc, nf, N_samples=S, N_importance=NI, moves=moved, chunk=CHUNK, device=dev)
    with torch.no_grad():
        ms = alternate({"edited_grid+grid_view(moves)": preview, "render_moves+render_frame": render}, a.reps, a.warmup,
                       clock=host_ms)
        e_occ, e_labels, _ = OB.edited_grid(occ, labels, T, moves, EXT, level)
        moved = OB.render_moves(occ, labels, T, moves, EXT, level, near, far, NI)
        o, d = get_rays_k(H, W, K, pose)

        def query(cr):
            cast, (move, point, vdir) = cr
            hit = cast["hit"]
            return mlp_forward_points(nf, point[hit], (vdir / torch.norm(vdir, dim=-1, keepdim=True))[hit])
        stages = []
        for r in range(a.warmup + a.reps):
            t, res = stages_ms(lambda: OB.cast_grid(e_occ, e_labels, T, o, d, near, far, EXT, level),
                               lambda cast: (cast, OB._edit_view(e_occ, e_labels, moved, source, o, d, cast)), query)
            if r >= a.warmup:
                stages.append(t)
        moved_px = int((res[1][1][0] >= 0).sum())
    med = {k2: _med(v) for k2, v in ms.items()}
    st = np.asarray(stages)
    return {"moves": n_moves, "labels": [k2 for k2, _ in moves], "moved_pixels": moved_px,
            "ms": {k2: [round(x, 2) for x in v] for k2, v in ms.items()}, "ms_median": med,
            "render_over_preview": round(med["render_moves+render_frame"] / med["edited_grid+grid_view(moves)"], 1),
            "device_ms_median": {"cast": _med(st[:, 0]), "replay": _med(st[:, 1]), "network": _med(st[:, 2])}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    dev = cuda_device("grid_view_bench.py")
    w = synth.workload("dmsr_study")
    H, W, K, ins_num = w["H"], w["W"], np.asarray(w["K"], dtype=np.float32), w["ins_num"]
    near, far = float(w["near"]), float(w["far"])
    pose = torch.as_tensor(np.asarray(w["c2w"], dtype=np.float32), device=dev)
    nc, nf, _, _ = make_models(101, 202, ins_num, dev)
    T = np.eye(4)
    out = {"bench": "grid_view", "workload": "dmsr_study", "ins_num": ins_num, "frame": "%dx%d" % (W, H), "reps": a.reps,
           "grid_view": []}
    for dim in (256, 512):
        with torch.no_grad():
            occ, labels = OB.occupancy_objects(nf, T, OB.object_mask(ins_num, remove=[]), dim, EXT, near, far, NI, device=dev)
        sample = occ.flatten()[::17]
        sample = sample[sample > 0]
        level = 0.45 if float(occ.min()) < 0.45 < float(occ.max()) else float(sample.kthvalue(int(0.9 * sample.numel())).values)
        view = lambda: OB.grid_view(occ, labels, T, H, W, K, pose, near, far, EXT, level)   # noqa: E731
        ms = alternate({"grid_view": view}, a.reps, a.warmup, clock=event_ms)["grid_view"]
        hits = int(view()["hit"].sum())
        rec = {"grid_dim": dim, "level": level, "hit_pixels": hits, "ms": [round(x, 3) for x in ms], "ms_median": _med(ms),
               "mrays_per_s": round(H * W / np.median(ms) / 1e3, 1)}
        rec["cast_kernel_ms"] = _kernel_ms(view)
        out["grid_view"].append(rec)
        if dim == 256:
            k, c = torch.unique(labels[occ > level], return_counts=True)
            label = int(k[torch.argmax(c)])
            A, _ = OB.grid_affine(T, dim, EXT)
            m = np.eye(4)
            m[:3, 3] = A @ np.asarray([8.0, 0.0, 0.0])
            moves = [(label, m)]

            def preview():
                e_occ, e_labels, _ = OB.edited_grid(occ, labels, T, moves, EXT, level)
                return OB.grid_view(e_occ, e_labels, T, H, W, K, pose, near, far, EXT, level)

            def render():
                moved = OB.render_moves(occ, labels, T, moves, EXT, level, near, far, NI)
                return render_frame(H, W, K, pose, near, far, nc, nf, N_samples=S, N_importance=NI, moves=moved, chunk=CHUNK,
                                    device=dev)
            with torch.no_grad():
                ms2 = alternate({"edited_grid+grid_view": preview, "render_moves+render_frame": render}, a.reps, a.warmup,
                                clock=host_ms)
            med = {k2: _med(v) for k2, v in ms2.items()}
            out["look"] = {"grid_dim": dim, "label": label, "ms": {k2: [round(x, 2) for x in v] for k2, v in ms2.items()},
                           "ms_median": med,
                           "render_over_preview": round(med["render_moves+render_frame"] / med["edited_grid+grid_view"], 1)}
            out["colour"] = [_colour(occ, labels, T, H, W, K, pose, near, far, level, nc, nf, dev, n, a) for n in (1, 3)]
        del occ, labels
    name, smi, card = gpu_identity(dev)
    name, power = card or (name, "unknown")
    out.update(gpu=name, power_limit=power, gpu_identity=smi)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
