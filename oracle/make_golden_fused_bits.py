"""Generate tests/golden/fused_bits.npz: the exact bits the fused render kernel and the RAW-mode training forward return on
seeded inputs, so that a change to the kernels' schedule can be held to bit identity with the commit that wrote the fixture.

Run on a GPU, with the commit whose results are to be pinned built in this tree:
    python oracle/make_golden_fused_bits.py [--out PATH]

Cases (the workloads bench.py times, networks of testing.make_models(101, 202), rays of synth.workload):
  * dmsr_study (ins_num 13) and replica_room0_93 (ins_num 93): 2048 rays spread over the frame, rendered through the single
    fused kernel (want_raw=False, want_samples=True) with want_coarse True and False, by the exact and the fp16 network;
  * the RAW-mode training forward (dmnerf_mlp_forward_train, exact network) on 1024 embedded samples of dmsr_study: its
    output and the saved activation planes.

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
N_RAYS = 2048
N_TRAIN = 1024
ROW_STRIDE = 64
WORKLOADS = ("dmsr_study", "replica_room0_93")


def render_cases(dev):
    """(name, tensor) for every array the fused-kernel cases return."""
    from dmnerf_b200 import _lib, synth
    from dmnerf_b200.render import render_rays
    from dmnerf_b200.testing import make_models
    for wname in WORKLOADS:
        wl = synth.workload(wname)
        sel = np.linspace(0, wl["H"] * wl["W"] - 1, N_RAYS).astype(np.int64)
        ro, rd = torch.from_numpy(wl["rays_o"][sel]).to(dev), torch.from_numpy(wl["rays_d"][sel]).to(dev)
        z = (torch.linspace(0, 1, 64) * (wl["far"] - wl["near"]) + wl["near"]).to(dev)
        nc, nf, _, _ = make_models(101, 202, wl["ins_num"], dev)
        for prec, impl in (("exact", _lib.IMPL_UMMA), ("f16", _lib.IMPL_UMMA_F16)):
            for want_coarse in (True, False):
                with torch.no_grad():
                    out = render_rays(ro, rd, nc, nf, z, want_raw=False, want_coarse=want_coarse, want_samples=True, impl=impl)
                tag = "%s/%s/%s" % (wname, prec, "coarse" if want_coarse else "fine_only")
                for k in sorted(out.keys()):
                    yield "%s/%s" % (tag, k), out[k]


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


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), dtype=np.uint8)


def rows(a):
    return np.ascontiguousarray(a[::ROW_STRIDE]) if a.ndim else a


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=OUT)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the fixture is the GPU kernels' output"
    dev = "cuda:0"
    save = {}
    for gen in (render_cases(dev), train_cases(dev)):
        for name, t in gen:
            a = t.detach().cpu().numpy()
            save[name + "#sha256"] = digest(a)
            save[name + "#shape"] = np.array(a.shape, dtype=np.int64)
            save[name + "#dtype"] = np.array(str(a.dtype))
            save[name + "#rows"] = rows(a)
    save["card"] = np.array(torch.cuda.get_device_name(0))
    np.savez_compressed(args.out, **save)
    print("wrote %s: %d arrays (%.1f KB)" % (args.out, len(save) // 4, os.path.getsize(args.out) / 1024))


if __name__ == "__main__":
    main()
