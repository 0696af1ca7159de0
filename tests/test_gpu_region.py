"""Region selection on the GPU (DESIGN.md, "Region selection"): the builders against scipy, the per-point test against its numpy
twin, identity and emptiness of trivial regions on every render path, the exclusion the oracle restates, rejections, and the
render_objects tool's piece flags."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from dmnerf_b200 import _lib, synth
from dmnerf_b200 import objects as OB
from dmnerf_b200.engine import get_context
from dmnerf_b200.render import render_frame, render_rays
from dmnerf_b200.testing import make_models, max_rel_err
from oracle import dmnerf_f16 as H
from oracle import dmnerf_oracle as O
from oracle import inventory_oracle as IO
from oracle import objects_oracle as OO
from oracle import region_oracle as RO

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
MAPS = ("rgb_coarse", "depth_coarse", "acc_coarse", "ins_coarse", "rgb_fine", "depth_fine", "acc_fine", "ins_fine")


def _rays(name, n, first=0):
    wl = synth.workload(name)
    sel = np.linspace(first, wl["H"] * wl["W"] - 1, n).astype(np.int64)
    return wl, torch.from_numpy(wl["rays_o"][sel]).to(DEV).contiguous(), torch.from_numpy(wl["rays_d"][sel]).to(DEV).contiguous()


def _z(wl):
    return O.z_val_sample(1, wl["near"], wl["far"], 64)[0].to(DEV)


def _equal(a, b, keys):
    for k in keys:
        assert torch.equal(a[k], b[k]), k


def _transform():
    T = np.eye(4)
    T[:3, 3] = (0.1, -0.2, 0.3)
    return T


def _bits_np(region):
    return region.bits.cpu().numpy().view(np.uint32)


# ------------------------------------------------------------------------------------------ builders against scipy
def _grids(dim):
    rng = np.random.default_rng(dim)
    blobs = np.zeros((dim,) * 3, dtype=bool)
    for _ in range(6):                                       # boxes of assorted sizes, as the components tests draw
        lo = rng.integers(0, dim - 2, 3)
        hi = np.minimum(lo + rng.integers(1, max(2, dim // 5), 3), dim)
        blobs[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] = True
    sparse = rng.random((dim,) * 3) < 0.002
    i, j, k = np.indices((dim,) * 3)
    checker = (i + j + k) % 2 == 0
    corners = np.zeros((dim,) * 3, dtype=bool)
    for c in range(8):
        corners[tuple((dim - 1) * ((c >> a) & 1) for a in range(3))] = True
    out = {"blobs": blobs | sparse, "corners": corners, "empty": np.zeros((dim,) * 3, dtype=bool),
           "full": np.ones((dim,) * 3, dtype=bool)}
    if dim < 256:
        out["checker"] = checker
    return out


@pytest.mark.parametrize("dim", [64, 97, 256])
def test_pack_and_dilate_equal_scipy(dim):
    T = _transform()
    for name, mask in _grids(dim).items():
        m = torch.from_numpy(mask).to(DEV)
        for conn in (6, 26):
            want = mask
            for r in range(4):
                if r:
                    want = RO.dilate(want, 1, conn)                 # r steps of one = scipy's iterations=r, zero border
                reg = OB.region_from_mask(m, T, dilate=r, connectivity=conn)
                got = _bits_np(reg)
                assert np.array_equal(got, RO.pack(want)), (name, conn, r)
                if r == 1 and name == "blobs":
                    inv = OB._region_bits(torch.where(m, 0, -1).int(), [1], 1, dim, r, conn, True)
                    assert np.array_equal(inv.cpu().numpy().view(np.uint32), RO.pack(~want)), (name, conn, "invert")
    # pack through component ids: a table over ids, -1 and ids past the table give 0
    rng = np.random.default_rng(1)
    ids = rng.integers(-1, 40, (dim,) * 3).astype(np.int32)
    chosen = [0, 3, 31, 32, 39]
    cc = {"grid": torch.from_numpy(ids).to(DEV), "label": np.arange(40, dtype=np.int16) % 5, "voxels": np.ones(40, dtype=np.int64)}
    reg = OB.component_region(cc, chosen, T, dilate=0)
    assert np.array_equal(_bits_np(reg), RO.pack_ids(ids, chosen))
    assert reg.applies == OB.label_words(sorted({c % 5 for c in chosen}))
    get_context(DEV).sync_check()


# ------------------------------------------------------------------------------------------ the per-point test
def test_region_contains_equals_the_twin():
    rng = np.random.default_rng(2)
    T, ext = _transform(), (1.9, 7.0, 7.0)
    for dim in (64, 97, 256):
        mask = rng.random((dim,) * 3) < 0.5
        reg = OB.region_from_mask(torch.from_numpy(mask).to(DEV), T, ext)
        idx = rng.integers(0, dim, (200000, 3))
        pts = [IO.grid_points_fp32(idx, T, dim, ext)]
        A, b = OB.grid_affine(T, dim, ext)
        pts.append(((rng.random((200000, 3)) * 1.2 - 0.1) * (dim - 1)) @ A.T + b)          # inside and around the grid
        pts.append(np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf]]) + b)
        pts = np.concatenate(pts).astype(np.float32)
        got = OB.region_contains(reg, torch.from_numpy(pts).to(DEV)).cpu().numpy()
        want = RO.contains(reg.voxel_map, _bits_np(reg), dim, pts)
        assert np.array_equal(got, want), (dim, int((got != want).sum()))
        assert want[:200000].tolist() == mask[idx[:, 0], idx[:, 1], idx[:, 2]].tolist()
    # half-index boundaries: a map [I | 0], points on k + 0.5 and near it; rint is half to even
    dim = 16
    vm = np.concatenate([np.eye(3), np.zeros((3, 1))], 1).astype(np.float32)
    mask = rng.random((dim,) * 3) < 0.5
    reg = OB.Region(OB.region_from_mask(torch.from_numpy(mask).to(DEV), T).bits, dim, vm)
    k = np.arange(-2, dim + 1, dtype=np.float32) + 0.5
    g = np.stack(np.meshgrid(k, k, k, indexing="ij"), -1).reshape(-1, 3)
    g = np.concatenate([g, np.nextafter(g, np.float32(np.inf)), np.nextafter(g, np.float32(-np.inf)),
                        rng.random((20000, 3)).astype(np.float32) * (dim + 2) - 1.5]).astype(np.float32)
    got = OB.region_contains(reg, torch.from_numpy(g).to(DEV)).cpu().numpy()
    assert np.array_equal(got, RO.contains(vm, _bits_np(reg), dim, g))


# ------------------------------------------------------------------------------------------ trivial regions
def _all(dim, value, outside):
    bits = torch.full(((dim ** 3 + 31) // 32,), -1 if value else 0, dtype=torch.int32, device=DEV)
    if value and dim ** 3 % 32:
        bits[-1] = (1 << (dim ** 3 % 32)) - 1
    return OB.Region(bits, dim, OB.voxel_map(_transform(), dim), None, outside)


@pytest.mark.parametrize("ins_num", [1, 13, 93, 127])
def test_all_ones_region_is_the_identity(ins_num):
    wl, ro, rd = _rays("dmsr_study", 513)
    nc, nf, _, _ = make_models(101, 202, ins_num, DEV)
    ones = _all(33, True, "keep")
    kept = [k for k in range(ins_num + 1) if k % 3 != 1]
    with torch.no_grad():
        for impl in (_lib.IMPL_AUTO, _lib.IMPL_UMMA_F16):
            for sel in (None, kept):
                kw = dict(want_raw=False, want_samples=True, impl=impl, keep_objects=sel)
                _equal(render_rays(ro, rd, nc, nf, _z(wl), **kw), render_rays(ro, rd, nc, nf, _z(wl), region=ones, **kw),
                       MAPS + ("weights_fine", "z_vals_fine"))
        for impl in (_lib.IMPL_SIMT, _lib.IMPL_UMMA):                      # the stage path: want_raw, SIMT and tensor-core
            a = render_rays(ro, rd, nc, nf, _z(wl), impl=impl)
            _equal(a, render_rays(ro, rd, nc, nf, _z(wl), impl=impl, region=ones), a.keys())
        K, c2w = wl["K"], wl["c2w"]
        fa = render_frame(wl["H"], wl["W"], K, c2w, wl["near"], wl["far"], nc, nf, pixel_range=(100001, 513), device=DEV)
        fb = render_frame(wl["H"], wl["W"], K, c2w, wl["near"], wl["far"], nc, nf, pixel_range=(100001, 513), device=DEV, region=ones)
        _equal(fa, fb, fa.keys())
    get_context(DEV).sync_check()


@pytest.mark.parametrize("impl", [_lib.IMPL_AUTO, _lib.IMPL_UMMA_F16, _lib.IMPL_SIMT])
def test_all_zero_region_dropping_everything_is_empty(impl):
    wl, ro, rd = _rays("replica_room0", 300)
    nc, nf, _, _ = make_models(101, 202, wl["ins_num"], DEV)
    zero = _all(20, False, "drop")
    with torch.no_grad():
        e = render_rays(ro, rd, nc, nf, _z(wl), impl=impl, want_raw=impl == _lib.IMPL_SIMT, region=zero)
    for s in ("coarse", "fine"):
        for k in ("rgb_", "depth_", "acc_"):
            assert bool((e[k + s] == 0).all()), k + s
        assert bool((e["ins_" + s] == 0.5).all())


# ------------------------------------------------------------------------------------------ regions of a labelled sweep
def _pieces(nf, ins_num, dim=64):
    T = _transform()
    with torch.no_grad():
        occ, lab = OB.occupancy_objects(nf, T, OB.object_mask(ins_num, keep=range(ins_num)), dim, device=DEV)
        sample = occ.flatten()
        level = float(sample.kthvalue(int(0.9 * sample.numel())).values)
        cc = OB.object_components(occ, lab, level, 26)
    best = OB.largest_components(cc["label"], cc["voxels"])
    biggest = int(np.argmax(cc["voxels"]))
    other = [c for c in range(len(cc["voxels"])) if int(cc["label"][c]) == int(cc["label"][biggest]) and c != biggest]
    return T, cc, {
        "drop_largest": OB.component_region(cc, [biggest], T, dilate=0, invert=True),
        "keep_one": OB.component_region(cc, [other[0] if other else biggest], T, dilate=1),
        "floaters": OB.component_region(cc, [best[k] for k in sorted(best) if k != ins_num], T, dilate=1)}


def _excluded(region, ins_num, ro, rd, z, raw):
    ex = RO.exclusion(region.voxel_map, _bits_np(region), region.dim, region.applies_words(ins_num), region.outside == "keep",
                      ro.cpu().numpy(), rd.cpu().numpy())
    return ex(z.cpu(), OO.object_labels(raw.cpu()))


@pytest.mark.parametrize("name,ins_num", [("dmsr_study", 13), ("replica_room0_93", 93)])
def test_component_regions_exclude_what_the_oracle_excludes(name, ins_num):
    """Stage path: every sample the oracle's rule excludes, on the kernels' own depths and network outputs, has weight exactly 0,
    and the weights elsewhere are the unselected composite's on those samples.  Fused path (exact and fp16): the same decisions
    on its own depths wherever the label is not a near tie, and the frame driver equals render_rays with the region."""
    wl, ro, rd = _rays(name, 1024)
    nc, nf, _, _ = make_models(101, 202, ins_num, DEV)
    T, cc, regions = _pieces(nf, ins_num)
    from dmnerf_b200.autograd import mlp_forward_rays
    hit = 0
    with torch.no_grad():
        for tag, reg in regions.items():
            for impl in (_lib.IMPL_SIMT, _lib.IMPL_UMMA):
                out = render_rays(ro, rd, nc, nf, _z(wl), impl=impl, region=reg)
                for p in ("coarse", "fine"):
                    ex = _excluded(reg, ins_num, ro, rd, out["z_vals_" + p], out["raw_" + p])
                    hit += int(ex.sum())
                    assert bool((out["weights_" + p].cpu()[ex] == 0).all()), (tag, impl, p)
                    want = O.composite(RO.exclude_samples(out["raw_" + p].cpu().double(), ex), out["z_vals_" + p].cpu().double(),
                                       rd.cpu().double())
                    # rays without a near-tied label (where fp32 sigmoids of host and device could pick another first maximum)
                    top = torch.topk(torch.sigmoid(out["raw_" + p][..., 4:].cpu().double()), 2, -1).values
                    ok = ((top[..., 0] - top[..., 1]) > 1e-5).all(-1)
                    err = (out["weights_" + p].cpu().double() - want[1]).abs()[ok]
                    assert float(err.max()) <= 1e-5, (tag, impl, p)
            for impl in (_lib.IMPL_AUTO, _lib.IMPL_UMMA_F16):
                out = render_rays(ro, rd, nc, nf, _z(wl), want_raw=False, want_samples=True, impl=impl, region=reg)
                for p, net, S in (("coarse", nc, 64), ("fine", nf, 192)):
                    z = out["z_vals_" + p] if p == "fine" else out["z_vals_coarse"]
                    raw = mlp_forward_rays(net, ro, rd, z.contiguous()).reshape(ro.shape[0], S, -1)
                    ex = _excluded(reg, ins_num, ro, rd, z, raw)
                    top = torch.topk(torch.sigmoid(raw[..., 4:].double()), 2, -1).values.cpu()
                    clear = (top[..., 0] - top[..., 1]) > (2e-2 if impl == _lib.IMPL_UMMA_F16 else 1e-3)
                    assert bool((out["weights_" + p].cpu()[ex & clear] == 0).all()), (tag, impl, p)
            # the frame driver with a pixel range against render_rays on the same rays and depths
            from dmnerf_b200.helpers import get_rays_k, z_val_sample
            H, W = wl["H"], wl["W"]
            c2w = torch.from_numpy(np.asarray(wl["c2w"], dtype=np.float32))
            fr = render_frame(H, W, wl["K"], c2w, wl["near"], wl["far"], nc, nf, pixel_range=(150001, 777), device=DEV, region=reg)
            fro, frd = get_rays_k(H, W, wl["K"], c2w.to(DEV))
            sl = slice(150001, 150001 + 777)
            ref = render_rays(fro.reshape(-1, 3)[sl], frd.reshape(-1, 3)[sl], nc, nf,
                              z_val_sample(777, wl["near"], wl["far"], 64, device=DEV), want_raw=False, region=reg)
            for k in ("rgb", "depth", "acc", "ins"):
                assert torch.equal(fr[k], ref[k + "_fine"].cpu()), (tag, k)
    assert hit > 0
    get_context(DEV).sync_check()


# ------------------------------------------------------------------------------------------ fused maps, teacher-forced
# As test_gpu_preview_edges.test_selected_render_teacher_forced: T is the fp16 restatement, E the fp64 network, both on the
# kernel's fp32 inputs at the kernel's own depths, composited in fp64 with the region's exclusion (region_oracle.render_on_depths).
FP16_TWIN_FRACTION = 0.3
FLOORS = {"rgb": 1e-2, "depth": 1e-1, "acc": 1e-2, "ins": 1e-2, "weights": 1.0}
_TF = {}


def _tf_setup(ins_num):
    """(nc, nf, oracle networks, regions of the labelled sweep) of one head width, built once per module."""
    if ins_num not in _TF:
        nc, nf, wc, wf = make_models(101, 202, ins_num, DEV)
        nets = {}
        for tag, w in (("coarse", wc), ("fine", wf)):
            p32 = {k: v.to(DEV) for k, v in O.to_torch(w).items()}
            p64 = {k: v.to(DEV) for k, v in O.to_torch(w, torch.float64).items()}
            nets[tag, "T"] = lambda x, p=p32: H.mlp_forward_f16(p, x.to(DEV)).cpu()
            nets[tag, "E"] = lambda x, p=p64: O.mlp_forward(p, x.to(DEV).double()).cpu()
        _TF[ins_num] = (nc, nf, nets, _pieces(nf, ins_num)[2])
    return _TF[ins_num]


@pytest.mark.parametrize("tag", ["drop_largest", "keep_one", "floaters"])
@pytest.mark.parametrize("ins_num", [13, 93])
@pytest.mark.parametrize("impl", [pytest.param(_lib.IMPL_UMMA, id="exact"), pytest.param(_lib.IMPL_UMMA_F16, id="f16")])
def test_fused_region_maps_teacher_forced(impl, ins_num, tag):
    """The fused kernel with a region of the labelled sweep on 513 rays: every map and weight of both passes against E (exact:
    1e-4 with a floor of a tenth of each map's scale) or within FP16_TWIN_FRACTION of T's distance to E (fp16, plus 4x the
    distance of an fp32 composite of T's own raw), on the kernel's own depths.  A ray is set aside only where a label that
    matters is ambiguous (the reference's two largest sigmoids closer than 4x the kernel-reference sigmoid difference): at most
    1 % of the rays for the exact network, 4 % for fp16, as for object selection."""
    from dmnerf_b200.autograd import mlp_forward_rays
    f16 = impl == _lib.IMPL_UMMA_F16
    nc, nf, nets, regions = _tf_setup(ins_num)
    reg = regions[tag]
    wl, ro, rd = _rays("dmsr_study", 513)
    with torch.no_grad():
        got = render_rays(ro, rd, nc, nf, _z(wl), want_raw=False, want_samples=True, impl=impl, region=reg)
        logits = {p: mlp_forward_rays(net, ro, rd, got["z_vals_" + p].contiguous(), impl).cpu().double()
                  for p, net in (("coarse", nc), ("fine", nf))}
    get_context(DEV).sync_check()
    ex = RO.exclusion(reg.voxel_map, _bits_np(reg), reg.dim, reg.applies_words(ins_num), reg.outside == "keep",
                      ro.cpu().numpy(), rd.cpu().numpy())
    roc, rdc = ro.cpu(), rd.cpu()
    zs = {p: got["z_vals_" + p].cpu() for p in ("coarse", "fine")}
    refs = {r: RO.render_on_depths(nets["coarse", r], nets["fine", r], roc, rdc, zs["coarse"], zs["fine"], exclude=ex)
            for r in ("T", "E")}
    R = refs["T" if f16 else "E"]
    n = ro.shape[0]
    ambiguous = torch.zeros(n, dtype=torch.bool)
    excluded = 0
    for p in ("coarse", "fine"):
        lg = logits[p].reshape(R["raw_" + p].shape)
        diff = (torch.sigmoid(lg[..., 4:]) - torch.sigmoid(R["raw_" + p][..., 4:])).abs().amax(-1)
        trans = 1.0 - torch.cumsum(R["weights_" + p], -1) + R["weights_" + p]
        matters = (R["raw_" + p][..., 3] > 0) & (trans > 1e-6)
        ambiguous |= ((R["gap_" + p] < 4.0 * diff) & matters).any(-1)
        excluded += int((ex(zs[p], R["labels_" + p]) & matters).sum())
    n_aside = int(ambiguous.sum())
    print("\n  region %s ins_num %d %s: %d excluded samples that matter, %d rays set aside" % (
        "f16" if f16 else "exact", ins_num, tag, excluded, n_aside))
    assert excluded > 0                                   # the region changes these renders
    assert n_aside <= (0.04 if f16 else 0.01) * n, n_aside
    keep = ~ambiguous
    for p in ("coarse", "fine"):
        if f16:
            T, E = refs["T"], refs["E"]
            raw32 = RO.exclude_samples(T["raw_" + p], ex(zs[p], T["labels_" + p])).float()
            t32 = dict(zip(("rgb", "weights", "depth", "ins", "acc"), O.composite(raw32, zs[p].float(), rdc.float())))
        for m in ("rgb", "depth", "acc", "ins", "weights"):
            k = "%s_%s" % (m, p)
            K = got[k].cpu().double()[keep]
            if f16:
                k_t, t_e = H.rel_l2(K, T[k][keep]), H.rel_l2(T[k][keep], E[k][keep])
                floor = H.rel_l2(t32[m].double()[keep], T[k][keep])
                print("    %-16s K-T %.2e  T-E %.2e  ratio %.3f" % (k, k_t, t_e, k_t / max(t_e, 1e-300)))
                assert k_t <= FP16_TWIN_FRACTION * t_e + 4.0 * floor, (k, k_t, t_e, floor)
            else:
                ref = R[k][keep].numpy()
                e = max_rel_err(K.numpy(), ref, max(FLOORS[m], 0.1 * float(np.abs(ref).max())))
                print("    %-16s max rel err %.2e" % (k, e))
                assert e <= 1e-4, (k, e)


# ------------------------------------------------------------------------------------------ rejections
def test_rejections():
    wl, ro, rd = _rays("dmsr_study", 64)
    nc, nf, _, _ = make_models(101, 202, 13, DEV)
    ctx = get_context(DEV)
    ctx.bind(0, nc); ctx.bind(1, nf)
    lib, st, n = ctx.lib, ctx.stream(), ro.shape[0]
    z, out = _z(wl), torch.empty(n, 3, device=DEV)
    with torch.no_grad():
        plain = render_rays(ro, rd, nc, nf, z, want_raw=False, want_samples=False)["rgb_fine"]
    io = _lib.RenderIO(rays_o=ro.data_ptr(), rays_d=rd.data_ptr(), z_coarse=z.data_ptr(), rgb_fine=out.data_ptr())
    words = torch.zeros(16, dtype=torch.int32, device=DEV)

    def render(desc, flags=0):
        edit = _lib.Edit(region=C.pointer(desc))
        io.edit = C.pointer(edit)
        return lib.dmnerf_render_forward(ctx.handle, io, n, 64, 128, flags, 0, st)
    good = OB.Region(words, 8, OB.voxel_map(_transform(), 8))
    # a region without bits, dim out of range, a non-finite map, applies above ins_num (naming the label)
    desc = good.abi(13)
    desc.bits = None
    assert render(desc) != 0 and b"NULL bits" in lib.dmnerf_last_error()
    for dim in (1, 1291):
        desc = good.abi(13)
        desc.dim = dim
        assert render(desc) != 0 and b"dim" in lib.dmnerf_last_error()
    desc = good.abi(13)
    desc.voxel_map[0] = float("nan")
    assert render(desc) != 0 and b"not finite" in lib.dmnerf_last_error()
    reg = OB.Region(words, 8, OB.voxel_map(_transform(), 8), applies=OB.label_words([2, 14]))
    assert render(reg.abi(13)) != 0 and b"applies to label 14, outside [0, 13]" in lib.dmnerf_last_error()
    # the flags that once selected the context's edits: rejected, not ignored
    io.edit = None
    for flag in (8, 16, 32):
        assert lib.dmnerf_render_forward(ctx.handle, io, n, 64, 128, flag, 0, st) != 0
        assert b"unknown flag" in lib.dmnerf_last_error()
    with torch.no_grad(), pytest.raises(RuntimeError, match="applies to label 14, outside \\[0, 13\\]"):
        render_rays(ro, rd, nc, nf, z, region=reg)
    with torch.no_grad(), pytest.raises(RuntimeError, match="applies to label 14"):
        render_frame(48, 64, wl["K"], wl["c2w"], 4.0, 15.0, nc, nf, device=DEV, region=reg)
    # bits of the wrong length, dtype or device
    for bits in (torch.zeros(17, dtype=torch.int32, device=DEV), torch.zeros(16, dtype=torch.int64, device=DEV),
                 torch.zeros(16, dtype=torch.int32)):
        with pytest.raises(ValueError):
            OB.Region(bits, 8, OB.voxel_map(_transform(), 8))
    # the autograd path
    with pytest.raises(RuntimeError, match="inference-only"):
        render_rays(ro, rd, nc, nf, z, region=OB.Region(words, 8, OB.voxel_map(_transform(), 8)))
    mask = torch.ones(8, 8, 8, dtype=torch.bool, device=DEV)
    for kw in ({"dilate": -1}, {"connectivity": 8}):
        with pytest.raises(ValueError):
            OB.region_from_mask(mask, _transform(), **kw)
    assert lib.dmnerf_region_dilate(ctx.handle, C.c_void_p(words.data_ptr()), 8, -1, 26, 0, C.c_void_p(out.data_ptr()), st) != 0
    assert lib.dmnerf_region_dilate(ctx.handle, C.c_void_p(words.data_ptr()), 8, 1, 18, 0, C.c_void_p(out.data_ptr()), st) != 0
    # a render with a region leaves nothing behind: the next render without an edit is the unselected one, bit for bit
    _lib.check(render(good.abi(13)), "dmnerf_render_forward")
    io.edit = None
    _lib.check(lib.dmnerf_render_forward(ctx.handle, io, n, 64, 128, 0, 0, st), "dmnerf_render_forward")
    assert torch.equal(out, plain)
    ctx.sync_check()


# ------------------------------------------------------------------------------------------ the tool
@pytest.mark.parametrize("flags", [["--no-floaters"], ["--drop-piece", "0"]])
def test_render_objects_tool_pieces(tmp_path, flags):
    nc, nf, _, _ = make_models(7, 8, 13, "cpu")
    ck = str(tmp_path / "ck.tar")
    torch.save({"network_coarse_state_dict": nc.state_dict(), "network_fine_state_dict": nf.state_dict()}, ck)
    wl = synth.workload("dmsr_study")
    H, W = 48, 64
    K = synth.dmsr_intrinsics(H, W)
    np.save(str(tmp_path / "pose.npy"), wl["c2w"])
    np.savetxt(str(tmp_path / "T.txt"), _transform())
    out = str(tmp_path / "out")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "render_objects.py"), ck, "--pose", str(tmp_path / "pose.npy"),
                        "--hwk", str(H), str(W)] + [repr(float(v)) for v in K.reshape(-1)] +
                       flags + ["--transform", str(tmp_path / "T.txt"), "--grid-dim", "48", "--level", "0.0", "--out", out],
                       capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["frames"] == 1 and sorted(os.listdir(out)) == ["000.png", "instance_000.png"]
