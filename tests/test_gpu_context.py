"""GPU: a context owns the device memory of its entry points.  Destroying it gives back everything they allocated, the
tensor-core backward's GEMM scratch included, however large a batch made it grow."""
import ctypes as C

import numpy as np
import pytest
import torch

from dmnerf_b200 import _lib, synth
from dmnerf_b200.engine import ordered_params
from dmnerf_b200.testing import make_models

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
N_RAYS, DIM, INS = 256, 32, 13


def _buffers(m):
    """Every tensor a cycle reads or writes, allocated before it runs: the cycle itself allocates nothing through torch."""
    e = lambda *shape, dtype=torch.float32: torch.zeros(shape, device=DEV, dtype=dtype)
    c, n3, f = 4 + INS + 1, DIM ** 3, 64 + 128
    wl = synth.workload("dmsr_study")
    sel = np.linspace(0, wl["H"] * wl["W"] - 1, N_RAYS).astype(np.int64)
    g = torch.Generator().manual_seed(7)
    idx = torch.stack(torch.meshgrid(*[torch.arange(DIM, dtype=torch.float32)] * 3, indexing="ij"))
    solid = ((idx - DIM / 2) ** 2).sum(0) < (DIM / 3) ** 2                       # a ball, two labels split at i = DIM / 2
    b = dict(
        ro=torch.as_tensor(wl["rays_o"][sel]).to(DEV), rd=torch.as_tensor(wl["rays_d"][sel]).to(DEV),
        z=torch.linspace(wl["near"], wl["far"], 64).to(DEV), raw_c=e(N_RAYS, 64, c), raw_f=e(N_RAYS, f, c), rgb=e(N_RAYS, 3),
        x=(torch.randn(m, 90, generator=g) * 0.5).to(DEV), out=e(m, c), acts=e(m * _lib.load().dmnerf_act_floats_per_sample()),
        d_out=(torch.randn(m, c, generator=g) * 1e-3).to(DEV), scratch=e(_lib.load().dmnerf_mlp_backward_scratch_floats(m)),
        occ_sweep=e(n3), lab_sweep=e(n3, dtype=torch.int16),
        occ=solid.float().reshape(-1).to(DEV), labels=(idx[0] >= DIM / 2).to(torch.int16).reshape(-1).to(DEV),
        verts=e(3 * n3, 3), tris=e(5 * n3, 3, dtype=torch.int32), normals=e(3 * n3, 3),
        cluster=e(5 * n3, dtype=torch.int32), csize=e(5 * n3, dtype=torch.int32),
        out_v=e(3 * n3, 3), out_n=e(3 * n3, 3), out_t=e(5 * n3, 3, dtype=torch.int32),
        comp=e(n3, dtype=torch.int32), c_label=e(n3, dtype=torch.int16), c_voxels=e(n3, dtype=torch.int64),
        c_root=e(n3, dtype=torch.int64), lut=e(n3, dtype=torch.int16), groups=e(n3, dtype=torch.int16),
        bits=torch.from_numpy(np.packbits(solid.numpy().reshape(-1), bitorder="little").view(np.int32)).to(DEV),
        dilated=e(n3 // 32, dtype=torch.int32))
    torch.cuda.synchronize()
    return b


def _cycle(params, grads, b, m):
    """One context through every entry point that allocates device scratch, then destroyed."""
    lib, st, p = _lib.load(), None, _lib.ptr
    h = C.c_void_p()
    _lib.check(lib.dmnerf_ctx_create(0, C.byref(h)), "dmnerf_ctx_create")
    call = lambda name, *args: _lib.check(getattr(lib, name)(h, *args, st), name)
    for slot in (0, 1):
        call("dmnerf_set_weights", slot, _lib.ptrs(params[slot]), len(params[slot]), INS)
    # the stage path (its depths and weights in context scratch), then the fp16 fused kernel
    io = _lib.RenderIO(rays_o=b["ro"].data_ptr(), rays_d=b["rd"].data_ptr(), z_coarse=b["z"].data_ptr(),
                       raw_coarse=b["raw_c"].data_ptr(), raw_fine=b["raw_f"].data_ptr(), rgb_fine=b["rgb"].data_ptr())
    call("dmnerf_render_forward", C.byref(io), N_RAYS, 64, 128, 0, _lib.IMPL_UMMA)
    io.raw_coarse = io.raw_fine = None
    call("dmnerf_render_forward", C.byref(io), N_RAYS, 64, 128, 0, _lib.IMPL_UMMA_F16)
    # the training network: forward with saved activations, backward through the tensor-core GEMMs
    call("dmnerf_mlp_forward_train", 1, p(b["x"]), None, None, None, m, 1, p(b["out"]), p(b["acts"]), _lib.IMPL_UMMA)
    call("dmnerf_mlp_backward", 1, p(b["acts"]), p(b["d_out"]), m, _lib.ptrs(grads), p(b["scratch"]), 3)
    # the mesh chain
    eye, ext = _lib.doubles(np.eye(4), 16), _lib.doubles([1.9, 7.0, 7.0], 3)
    keep = _lib.keep_mask([(1 << (INS + 1)) - 1, 0, 0, 0])
    call("dmnerf_mesh_occupancy", 1, eye, ext, DIM, 0.1, 0, keep, p(b["occ_sweep"]), p(b["lab_sweep"], torch.int16))
    counts = (C.c_int64 * 2)()
    call("dmnerf_mesh_mc_count", p(b["occ"]), DIM, DIM, DIM, 0.5, counts)
    nv, nt = counts[0], counts[1]
    assert nv > 0 and nt > 0
    call("dmnerf_mesh_mc_emit", p(b["occ"]), DIM, DIM, DIM, 0.5, p(b["verts"]), p(b["tris"], torch.int32))
    call("dmnerf_mesh_normals", p(b["verts"]), nv, p(b["tris"], torch.int32), nt, p(b["normals"]))
    call("dmnerf_mesh_clusters", p(b["tris"], torch.int32), nt, nv, p(b["cluster"], torch.int32), p(b["csize"], torch.int32))
    call("dmnerf_mesh_clean", p(b["verts"]), p(b["normals"]), nv, p(b["tris"], torch.int32), nt, p(b["csize"], torch.int32), 1,
         p(b["out_v"]), p(b["out_n"]), p(b["out_t"], torch.int32), counts)
    # the inventory, the connected components and a two-step dilation, on the labelled ball
    boxes = (C.c_int32 * 12)(*([0, DIM - 1] * 6))
    mom, hist, spans = (C.c_int64 * 20)(), (C.c_uint32 * (6 * DIM))(), (C.c_double * 12)()
    labels = p(b["labels"], torch.int16)
    call("dmnerf_object_voxels", p(b["occ"]), labels, DIM, 0.5, 2, boxes, mom, hist)
    call("dmnerf_object_spans", p(b["occ"]), labels, DIM, 0.5, 2, boxes, _lib.doubles(np.tile(np.eye(3, 4), (2, 1)), 24), spans)
    n_comp = C.c_int64()
    call("dmnerf_object_components", p(b["occ"]), labels, DIM, 0.5, 2, 26, p(b["comp"], torch.int32), C.byref(n_comp))
    assert n_comp.value >= 1
    call("dmnerf_component_table", p(b["comp"], torch.int32), labels, DIM, n_comp.value, p(b["c_label"], torch.int16),
         p(b["c_voxels"], torch.int64), p(b["c_root"], torch.int64))
    call("dmnerf_component_groups", p(b["comp"], torch.int32), DIM, n_comp.value, p(b["lut"], torch.int16), -1,
         p(b["groups"], torch.int16))
    call("dmnerf_region_dilate", p(b["bits"], torch.int32), DIM, 2, 6, 0, p(b["dilated"], torch.int32))
    call("dmnerf_sync_check")
    _lib.check(lib.dmnerf_ctx_destroy(h), "dmnerf_ctx_destroy")


def test_destroying_a_context_returns_its_device_memory():
    nc, nf, _, _ = make_models(101, 202, INS, DEV)
    params = [ordered_params(nc)[0], ordered_params(nf)[0]]
    grads = [torch.zeros_like(q) for q in params[1]]
    # warm-up on a context of its own: loads every module and sizes the local memory of every kernel the cycle launches
    _cycle(params, grads, _buffers(65536), 65536)
    big = _buffers(196608)
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    # the same cycle with a training batch three times as large: the backward's partial-product scratch grows with it
    _cycle(params, grads, big, 196608)
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    assert abs(free0 - free1) <= 2 << 20, "context destroyed, but %.1f MiB of device memory not returned" % ((free0 - free1) / 2**20)
