"""Parity of the TIMED kernel (the fused render kernel, render_rays(want_raw=False)) against the live CPU oracle on a few
thousand rays of every BASELINE config, with the oracle's own fp64 twin as the yard-stick.  Test infrastructure: imports
oracle/.  Writes gpurun_out/parity_at_scale.{json,md}.       python tools/parity_at_scale.py [n_rays]"""
import json
import os
import sys
import time

import numpy as np
import torch

from _harness import ROOT, cuda_device, gpu_identity
from dmnerf_b200 import synth
from dmnerf_b200.render import render_rays
from dmnerf_b200.testing import make_models, parity_table, format_parity_table
from dmnerf_b200.engine import get_context
from oracle import dmnerf_oracle as O

CONFIGS = ("dmsr_study", "replica_room0", "replica_room0_93", "replica_office2")


def run_config(name, n_rays, dev="cuda", seeds=(101, 202)):
    wl = synth.workload(name)
    sel = np.linspace(0, wl["H"] * wl["W"] - 1, n_rays).astype(np.int64)
    ro, rd = torch.from_numpy(wl["rays_o"][sel]), torch.from_numpy(wl["rays_d"][sel])
    nc, nf, wc, wf = make_models(seeds[0], seeds[1], wl["ins_num"], dev)
    z = O.z_val_sample(n_rays, wl["near"], wl["far"], 64)
    from dmnerf_b200 import _lib
    ctx = get_context(dev)
    ctx.bind(0, nc); ctx.bind(1, nf)                      # weight packing happens here, not inside the counted render call
    with torch.no_grad():
        before = _lib.launch_count()
        ours = render_rays(ro.to(dev), rd.to(dev), nc, nf, z[0].to(dev), want_raw=False, want_samples=False)
        launches = _lib.launch_count() - before
        ctx.sync_check()
        t0 = time.time()
        ref = O.render(ro, rd, O.to_torch(wc), O.to_torch(wf), z)
        t1 = time.time()
        twin = O.render(ro.double(), rd.double(), O.to_torch(wc, torch.float64), O.to_torch(wf, torch.float64),
                        O.z_val_sample(n_rays, wl["near"], wl["far"], 64, dtype=torch.float64))
    return parity_table(ours, twin, ref), {"oracle_s": t1 - t0, "twin_s": time.time() - t1, "n_rays": n_rays, "ins_num": wl["ins_num"],
                                          "render_launches": launches}


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 2048
    print("GPU: %s" % gpu_identity(cuda_device("parity_at_scale.py"))[1])
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    res, md = {}, []
    for name in CONFIGS:
        table, info = run_config(name, n)
        res[name] = {"table": table, "info": info}
        md.append(format_parity_table("%s (ins_num %d, %d rays)" % (name, info["ins_num"], n), table))
        print(md[-1], flush=True)
    json.dump(res, open(os.path.join(ROOT, "gpurun_out", "parity_at_scale.json"), "w"), indent=1)
    open(os.path.join(ROOT, "gpurun_out", "parity_at_scale.md"), "w").write("\n\n".join(md) + "\n")


if __name__ == "__main__":
    main()
