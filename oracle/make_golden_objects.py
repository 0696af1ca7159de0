"""Generate tests/golden/objects.npz: object-selected renders from the UNMODIFIED original `dm_nerf`, and pin the selection
oracle (oracle/objects_oracle.py) to them.

Run in the build container only (the original checkout does not exist on the GPU box):
    python oracle/make_golden_objects.py

The original has no object selection, so its networks are wrapped: `forward` returns the network output with the density
channel zeroed where the sample's label argmax(sigmoid(raw[..., 4:])) is not kept (objects_oracle.select_objects), and the
original's own dm_nerf renders with them.  objects_oracle.render must reproduce every map bit for bit.

Per workload (dmsr_study at ins_num 13, replica_room0 at ins_num 59; synthetic trained-like weights regenerated from their
seeds) and per selection (keep = {the label with the most fine weight}, remove = {that label}, the empty keep set) it stores
the maps, the weights, the fine depths and the per-sample coarse labels; for dmsr_study / remove also the unedited fine network
output of the first 8 rays, the input of the teacher-forced composite test.

Labels must be unambiguous in fp32: every stored sample (coarse and fine, every selection) is checked to have a gap of at least
1e-6 between its two largest instance sigmoids; the smallest gap found is recorded as `<tag>_min_gap`.
"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(1, "/root/reference")

from networks.render import dm_nerf as ref_dm_nerf                                     # noqa: E402
from networks.dm_nerf import get_embedder as ref_get_embedder, DM_NeRF as RefNet       # noqa: E402
from networks.helpers import z_val_sample as ref_z_val_sample                          # noqa: E402

torch.autograd.set_detect_anomaly(False)   # reference networks/dm_nerf.py:5 turns it on at import

from oracle import dmnerf_oracle as O   # noqa: E402
from oracle import objects_oracle as OO   # noqa: E402
from dmnerf_b200 import synth          # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "objects.npz")
MIN_GAP = 1e-6
N_TEACHER = 8


class Selected(torch.nn.Module):
    """The original network with the selection edit on its output; keeps the unedited output of the last call."""

    def __init__(self, net, keep):
        super().__init__()
        self.net, self.keep, self.last = net, keep, None

    def forward(self, x):
        raw = self.net(x)
        self.last = raw
        return OO.select_objects(raw, self.keep)


def ref_net(weights_np, ins_num):
    net = RefNet(8, 256, 63, 27, [4], ins_num)
    net.load_state_dict({k: torch.from_numpy(v) for k, v in weights_np.items()})
    return net


def same(a, b, what):
    if not torch.equal(a.detach(), b.detach()):
        raise SystemExit("oracle != original for %s (max abs diff %g)" % (what, (a - b).abs().max().item()))


def min_gap(raw):
    s = torch.sigmoid(raw[..., 4:].double()).reshape(-1, raw.shape[-1] - 4)
    top = torch.topk(s, 2, dim=-1).values
    return float((top[:, 0] - top[:, 1]).min())


def words(labels):
    w = [0, 0, 0, 0]
    for k in labels:
        w[k >> 5] |= 1 << (k & 31)
    return np.array(w, dtype=np.uint32)


def main():
    pe, _ = ref_get_embedder(10)
    ve, _ = ref_get_embedder(4)
    args = types.SimpleNamespace(perturb=0.0, N_importance=128, is_train=False, N_ins=None)
    save = {}
    # first pixel of the strided ray set: room0's set from pixel 0 holds a sample with a 9e-7 sigmoid gap, so it starts at 320
    for tag, wlname, ins_num, N, first in (("study", "dmsr_study", 13, 16, 0), ("room0", "replica_room0", 59, 8, 320)):
        wl = synth.workload(wlname)
        sel = np.linspace(first, wl["H"] * wl["W"] - 1, N).astype(np.int64)
        ro, rd = torch.from_numpy(wl["rays_o"][sel]), torch.from_numpy(wl["rays_d"][sel])
        wc, wf = synth.make_weights(101, ins_num), synth.make_weights(202, ins_num)
        zc = ref_z_val_sample(N, wl["near"], wl["far"], 64)
        with torch.no_grad():
            base = O.render(ro, rd, O.to_torch(wc), O.to_torch(wf), zc)
        mass = torch.zeros(ins_num + 1, dtype=torch.float64)
        mass.index_add_(0, OO.object_labels(base["raw_fine"]).reshape(-1), base["weights_fine"].double().reshape(-1))
        top = int(torch.argmax(mass))
        selections = {"keep": [top], "remove": [k for k in range(ins_num + 1) if k != top], "empty": []}
        gap = 1.0
        for name, kept in selections.items():
            keep = torch.zeros(ins_num + 1, dtype=torch.bool)
            keep[kept] = True
            nc, nf = Selected(ref_net(wc, ins_num), keep), Selected(ref_net(wf, ins_num), keep)
            with torch.no_grad():
                ref = ref_dm_nerf(torch.stack([ro, rd], 0), pe, ve, nc, nf, zc, args)
                mine = OO.render(ro, rd, O.to_torch(wc), O.to_torch(wf), zc, keep)
            for k in ("rgb_coarse", "rgb_fine", "depth_coarse", "depth_fine", "ins_coarse", "ins_fine", "z_vals_fine"):
                same(mine[k], ref[k], "%s/%s %s" % (tag, name, k))
            same(mine["raw_coarse"], nc.last.reshape(mine["raw_coarse"].shape), "%s/%s raw_coarse" % (tag, name))
            same(mine["raw_fine"], nf.last.reshape(mine["raw_fine"].shape), "%s/%s raw_fine" % (tag, name))
            gap = min(gap, min_gap(mine["raw_coarse"]), min_gap(mine["raw_fine"]))
            p = "%s_%s_" % (tag, name)
            save[p + "mask"] = words(kept)
            for k in ("rgb_coarse", "rgb_fine", "depth_coarse", "depth_fine", "ins_coarse", "ins_fine", "acc_coarse", "acc_fine",
                      "weights_coarse", "weights_fine", "z_vals_fine"):
                save[p + k] = mine[k].numpy()
            save[p + "labels_coarse"] = OO.object_labels(mine["raw_coarse"]).numpy().astype(np.int16)
            save[p + "labels_fine"] = OO.object_labels(mine["raw_fine"]).numpy().astype(np.int16)
            if tag == "study" and name == "remove":
                save[p + "raw_fine"] = mine["raw_fine"][:N_TEACHER].numpy()
        if gap < MIN_GAP:
            raise SystemExit("%s: a stored sample has a top-2 sigmoid gap of %g < %g: its label is ambiguous in fp32" % (tag, gap, MIN_GAP))
        save.update({tag + "_sel": sel, tag + "_rays_o": ro.numpy(), tag + "_rays_d": rd.numpy(), tag + "_near": wl["near"],
                     tag + "_far": wl["far"], tag + "_ins_num": ins_num, tag + "_min_gap": gap, tag + "_top": top})
        print("%s: ins_num %d, top label %d, min top-2 sigmoid gap %.3g" % (tag, ins_num, top, gap))
    save.update(seed_coarse=101, seed_fine=202)
    np.savez_compressed(OUT, **save)
    print("wrote %s (%.1f KB); oracle == original bit for bit on every selected render" % (OUT, os.path.getsize(OUT) / 1024))


if __name__ == "__main__":
    main()
