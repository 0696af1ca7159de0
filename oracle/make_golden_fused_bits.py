"""Generate tests/golden/fused_bits.npz and tests/golden/fused_edge_bits.npz: the exact bits the fused render kernels, the
RAW-mode training forward and a points-mode query return on seeded inputs, so that a change to the network kernel can be held
to bit identity with the commit that wrote the fixtures.

Run on a GPU, with the commit whose results are to be pinned built in this tree:
    python oracle/make_golden_fused_bits.py [--out PATH] [--edge-out PATH]

Cases (the workloads bench.py times, networks of testing.make_models(101, 202), rays of synth.workload).  fused_bits.npz:
  * dmsr_study (ins_num 13) and replica_room0_93 (ins_num 93): 2048 rays spread over the frame, rendered through the single
    fused kernel (want_raw=False, want_samples=True) with want_coarse True and False, by the exact and the fp16 network;
  * the RAW-mode training forward (dmnerf_mlp_forward_train, exact network) on 1024 embedded samples of dmsr_study: its
    output and the saved activation planes.
fused_edge_bits.npz:
  * the selected fused kernels on 1024 rays of dmsr_study, exact and fp16: one render with a keep mask, one with a region;
  * the same rays rendered at ins_num 1, 15, 16, 17 and 127, exact and fp16: the instance head's stage holds
    pad16(ins_num + 1) rows, and these widths sit on either side of each step of it;
  * a points-mode query (dmnerf_mlp_forward_points, exact and fp16) on 3001 points along rays of dmsr_study.

The arrays are too large to keep whole (well over 1 MB even compressed), so every array is stored as the SHA-256 of its raw
bytes with its shape and dtype, plus every 64th row of it in full, which says where a mismatch lies.
"""
import argparse
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

OUT = os.path.join(ROOT, "tests", "golden", "fused_bits.npz")
EDGE_OUT = os.path.join(ROOT, "tests", "golden", "fused_edge_bits.npz")
N_RAYS = 2048
N_SMALL = 1024                  # rays of the selected and the head-width renders
N_TRAIN = 1024
N_POINTS = 3001                 # not a multiple of the 128-row tile
HEAD_WIDTHS = (1, 15, 16, 17, 127)
ROW_STRIDE = 64
WORKLOADS = ("dmsr_study", "replica_room0_93")


def _rays(wname, n, dev):
    from dmnerf_b200 import synth
    wl = synth.workload(wname)
    sel = np.linspace(0, wl["H"] * wl["W"] - 1, n).astype(np.int64)
    ro, rd = torch.from_numpy(wl["rays_o"][sel]).to(dev), torch.from_numpy(wl["rays_d"][sel]).to(dev)
    z = (torch.linspace(0, 1, 64) * (wl["far"] - wl["near"]) + wl["near"]).to(dev)
    return wl, ro, rd, z


def _precisions():
    from dmnerf_b200 import _lib
    return (("exact", _lib.IMPL_UMMA), ("f16", _lib.IMPL_UMMA_F16))


def _render(tag, ro, rd, nc, nf, z, **kw):
    from dmnerf_b200.render import render_rays
    with torch.no_grad():
        out = render_rays(ro, rd, nc, nf, z, want_raw=False, want_samples=True, **kw)
    for k in sorted(out.keys()):
        yield "%s/%s" % (tag, k), out[k]


def render_cases(dev):
    """(name, tensor) for every array the fused-kernel cases of fused_bits.npz return."""
    from dmnerf_b200.testing import make_models
    for wname in WORKLOADS:
        wl, ro, rd, z = _rays(wname, N_RAYS, dev)
        nc, nf, _, _ = make_models(101, 202, wl["ins_num"], dev)
        for prec, impl in _precisions():
            for want_coarse in (True, False):
                tag = "%s/%s/%s" % (wname, prec, "coarse" if want_coarse else "fine_only")
                yield from _render(tag, ro, rd, nc, nf, z, want_coarse=want_coarse, impl=impl)


def edge_render_cases(dev):
    """(name, tensor) for every array the selected-kernel and head-width renders of fused_edge_bits.npz return."""
    from dmnerf_b200 import objects as OB
    from dmnerf_b200.testing import make_models
    # the selected kernels: a keep mask, and a region from a seeded voxel mask over the sweep grid (about a third of the fine
    # samples lie inside the grid).  These networks label the coarse samples 4, 10 or 13 and the fine samples 4, so the mask
    # drops the 10s: the coarse weights, hence the fine depths, change.
    wl, ro, rd, z = _rays("dmsr_study", N_SMALL, dev)
    nc, nf, _, _ = make_models(101, 202, wl["ins_num"], dev)
    keep = [k for k in range(wl["ins_num"] + 1) if k != 10]
    mask = torch.from_numpy(np.random.default_rng(7).random((64,) * 3) < 0.5).to(dev)
    region = OB.region_from_mask(mask, np.eye(4))
    for prec, impl in _precisions():
        yield from _render("dmsr_study/%s/keep" % prec, ro, rd, nc, nf, z, impl=impl, keep_objects=keep)
        yield from _render("dmsr_study/%s/region" % prec, ro, rd, nc, nf, z, impl=impl, region=region)
    # instance-head widths
    for ins_num in HEAD_WIDTHS:
        nc, nf, _, _ = make_models(101, 202, ins_num, dev)
        for prec, impl in _precisions():
            yield from _render("ins%d/%s" % (ins_num, prec), ro, rd, nc, nf, z, impl=impl)


def train_cases(dev):
    """(name, tensor) for the output and the saved planes of one RAW-mode training forward."""
    from dmnerf_b200 import _lib, synth
    from dmnerf_b200.engine import get_context
    from dmnerf_b200.testing import make_models
    from oracle import dmnerf_oracle as O
    wl = synth.workload("dmsr_study")
    sel = np.linspace(0, wl["H"] * wl["W"] - 1, N_TRAIN // 64).astype(np.int64)
    ro, rd = torch.from_numpy(wl["rays_o"][sel]), torch.from_numpy(wl["rays_d"][sel])
    z = O.z_val_sample(len(sel), wl["near"], wl["far"], 64)
    x, _ = O._net_inputs(ro, rd, rd / torch.linalg.norm(rd, dim=-1, keepdim=True), z)
    x = x.contiguous().float().to(dev)
    nc, _, _, _ = make_models(101, 202, wl["ins_num"], dev)
    ctx = get_context(dev)
    slot = ctx.slot_for(nc)
    ins_num = ctx.bind(slot, nc)
    m = x.shape[0]
    out = torch.zeros((m, 4 + ins_num + 1), device=dev, dtype=torch.float32)
    acts = torch.zeros(m * ctx.lib.dmnerf_act_floats_per_sample(), device=dev, dtype=torch.float32)
    ctx.call("dmnerf_mlp_forward_train", ctx.handle, slot, _lib.ptr(x), None, None, None, m, 1, _lib.ptr(out), _lib.ptr(acts),
             _lib.IMPL_UMMA)
    ctx.sync_check()
    yield "train/out", out
    yield "train/acts", acts.view(torch.int32)      # the planes hold ReLU bit words too: compare them as raw bits


def points_cases(dev):
    """(name, tensor) for a points-mode query of the exact and the fp16 network: points at seeded depths along rays of
    dmsr_study, with the rays' unit directions as view directions."""
    from dmnerf_b200.autograd import mlp_forward_points
    from dmnerf_b200.testing import make_models
    wl, ro, rd, _ = _rays("dmsr_study", N_POINTS, dev)
    t = torch.from_numpy(np.random.default_rng(11).uniform(wl["near"], wl["far"], (N_POINTS, 1)).astype(np.float32)).to(dev)
    pts = ro + rd * t
    vd = rd / torch.linalg.norm(rd, dim=-1, keepdim=True)
    nc, _, _, _ = make_models(101, 202, wl["ins_num"], dev)
    for prec, impl in _precisions():
        with torch.no_grad():
            yield "points/%s/out" % prec, mlp_forward_points(nc, pts, vd, impl=impl)


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), dtype=np.uint8)


def rows(a):
    return np.ascontiguousarray(a[::ROW_STRIDE]) if a.ndim else a


def write(path, gens):
    save = {}
    for gen in gens:
        for name, t in gen:
            a = t.detach().cpu().numpy()
            save[name + "#sha256"] = digest(a)
            save[name + "#shape"] = np.array(a.shape, dtype=np.int64)
            save[name + "#dtype"] = np.array(str(a.dtype))
            save[name + "#rows"] = rows(a)
    save["card"] = np.array(torch.cuda.get_device_name(0))
    np.savez_compressed(path, **save)
    print("wrote %s: %d arrays (%.1f KB)" % (path, len(save) // 4, os.path.getsize(path) / 1024))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=OUT)
    ap.add_argument("--edge-out", default=EDGE_OUT)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the fixture is the GPU kernels' output"
    dev = "cuda:0"
    write(args.out, (render_cases(dev), train_cases(dev)))
    write(args.edge_out, (edge_render_cases(dev), points_cases(dev)))


if __name__ == "__main__":
    main()
