"""Object appearance on the GPU (DESIGN.md, "Object appearance"): the identity table is the keep-all selected render bit for bit,
density 0 is removal bit for bit, a colour-only appearance changes rgb alone, the fused maps of an edited scene against the
teacher-forced oracle, rejections, and the render_objects tool's appearance flags."""
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
from oracle import appearance_oracle as AO
from oracle import dmnerf_f16 as H
from oracle import dmnerf_oracle as O
from oracle import objects_oracle as OO
from oracle import region_oracle as RO

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
MAPS = ("rgb_coarse", "depth_coarse", "acc_coarse", "ins_coarse", "rgb_fine", "depth_fine", "acc_fine", "ins_fine")
FUSED = MAPS + ("weights_coarse", "weights_fine", "z_vals_coarse", "z_vals_fine")


def _rays(name, n, first=0):
    wl = synth.workload(name)
    sel = np.linspace(first, wl["H"] * wl["W"] - 1, n).astype(np.int64)
    return wl, torch.from_numpy(wl["rays_o"][sel]).to(DEV).contiguous(), torch.from_numpy(wl["rays_d"][sel]).to(DEV).contiguous()


def _z(wl):
    return O.z_val_sample(1, wl["near"], wl["far"], 64)[0].to(DEV)


def _equal(a, b, keys, what=""):
    for k in keys:
        assert torch.equal(a[k], b[k]), (what, k)


def _floater_region(nf, ins_num, dim=64):
    """Every object label keeps its largest piece of a labelled sweep of the fine network (component_region)."""
    T = np.eye(4)
    T[:3, 3] = (0.1, -0.2, 0.3)
    with torch.no_grad():
        occ, lab = OB.occupancy_objects(nf, T, OB.object_mask(ins_num, keep=range(ins_num)), dim, device=DEV)
        sample = occ.flatten()
        level = float(sample.kthvalue(int(0.9 * sample.numel())).values)
        cc = OB.object_components(occ, lab, level, 26)
    best = OB.largest_components(cc["label"], cc["voxels"])
    return OB.component_region(cc, [best[k] for k in sorted(best) if k != ins_num], T, dilate=1)


def _paths(wl, ro, rd, nc, nf, **kw):
    """The renders of every path with the same edit arguments: fused exact and fp16 (with samples), the stage path with raw
    outputs (SIMT and tensor-core), and the frame driver on a pixel range."""
    out = {}
    for tag, impl in (("fused", _lib.IMPL_UMMA), ("fused_f16", _lib.IMPL_UMMA_F16)):
        out[tag] = render_rays(ro, rd, nc, nf, _z(wl), want_raw=False, want_samples=True, impl=impl, **kw)
    for tag, impl in (("simt", _lib.IMPL_SIMT), ("umma_raw", _lib.IMPL_UMMA)):
        out[tag] = render_rays(ro, rd, nc, nf, _z(wl), impl=impl, **kw)
    out["frame"] = render_frame(wl["H"], wl["W"], wl["K"], wl["c2w"], wl["near"], wl["far"], nc, nf, pixel_range=(100001, 513),
                                device=DEV, **kw)
    return out


def _compare(a, b, keys=None):
    for tag in a:
        _equal(a[tag], b[tag], keys[tag] if keys else a[tag].keys(), tag)


# ------------------------------------------------------------------------------------------ identity and removal
@pytest.mark.parametrize("ins_num", [1, 13, 93, 127])
def test_identity_is_the_keep_all_selection_and_density_zero_is_removal(ins_num):
    wl, ro, rd = _rays("dmsr_study", 513)
    nc, nf, _, _ = make_models(101, 202, ins_num, DEV)
    every = list(range(ins_num + 1))
    gone = [k for k in every if k % 3 == 1]
    with torch.no_grad():
        keep_all = _paths(wl, ro, rd, nc, nf, keep_objects=every)
        _compare(keep_all, _paths(wl, ro, rd, nc, nf, appearance=OB.Appearance(ins_num)))
        _compare(keep_all, _paths(wl, ro, rd, nc, nf, keep_objects=every, appearance=OB.Appearance(ins_num)))
        zero = OB.Appearance(ins_num, density={k: 0.0 for k in gone})
        removed = _paths(wl, ro, rd, nc, nf, keep_objects=[k for k in every if k not in gone])
        _compare(removed, _paths(wl, ro, rd, nc, nf, appearance=zero))
    get_context(DEV).sync_check()


@pytest.mark.parametrize("name,ins_num", [("dmsr_study", 13), ("replica_room0_93", 93)])
def test_density_zero_with_a_region_is_removal_with_that_region(name, ins_num):
    wl, ro, rd = _rays(name, 513)
    nc, nf, _, _ = make_models(101, 202, ins_num, DEV)
    reg = _floater_region(nf, ins_num)
    every = list(range(ins_num + 1))
    gone = [2, ins_num]
    kept = [k for k in every if k not in gone]
    with torch.no_grad():
        _compare(_paths(wl, ro, rd, nc, nf, keep_objects=kept, region=reg),
                 _paths(wl, ro, rd, nc, nf, region=reg, appearance=OB.Appearance(ins_num, density={k: 0 for k in gone})))
        _compare(_paths(wl, ro, rd, nc, nf, keep_objects=every, region=reg),
                 _paths(wl, ro, rd, nc, nf, region=reg, appearance=OB.Appearance(ins_num)))
    get_context(DEV).sync_check()


# ------------------------------------------------------------------------------------------ colour only
def _colour(ins_num):
    """A tint on the even labels, a channel swap with gain and offset (clamped) on the odd ones."""
    swap = np.array([[0.0, 0.0, 1.2, 0.05], [0.0, 1.0, 0.0, -0.1], [0.8, 0.0, 0.0, 0.0]])
    return {k: OB.tint((0.9, 0.25, 0.1)) if k % 2 == 0 else swap for k in range(ins_num + 1)}


@pytest.mark.parametrize("name,ins_num", [("dmsr_study", 13), ("replica_room0_93", 93)])
def test_colour_only_touches_rgb_alone(name, ins_num):
    """Every output but rgb is the keep-all selected render bit for bit; the stage path's rgb is the oracle composite of the
    kernel's own raw outputs and weights with the edited colours, on the rays without a near-tied label."""
    wl, ro, rd = _rays(name, 513)
    nc, nf, _, _ = make_models(101, 202, ins_num, DEV)
    app = OB.Appearance(ins_num, colour=_colour(ins_num))
    every = list(range(ins_num + 1))
    with torch.no_grad():
        base = _paths(wl, ro, rd, nc, nf, keep_objects=every)
        got = _paths(wl, ro, rd, nc, nf, appearance=app)
    for tag in base:
        keys = [k for k in base[tag] if not k.startswith("rgb")]
        _equal(base[tag], got[tag], keys, tag)
        rgb = [k for k in base[tag] if k.startswith("rgb")]
        assert rgb and all(not torch.equal(base[tag][k], got[tag][k]) for k in rgb), tag
    for tag in ("simt", "umma_raw"):
        out = got[tag]
        for p in ("coarse", "fine"):
            raw = out["raw_" + p].cpu()
            lab = OO.object_labels(raw)
            w, c = out["weights_" + p].cpu(), AO.edited_colour(raw, lab, app)
            want = torch.zeros(raw.shape[0], 3)
            for i in range(raw.shape[1]):                                  # the kernel's order: ascending samples, fp32
                want = want + w[:, i, None] * c[:, i]
            top = torch.topk(torch.sigmoid(raw[..., 4:].double()), 2, -1).values
            ok = ((top[..., 0] - top[..., 1]) > 1e-5).all(-1)
            err = float((out["rgb_" + p].cpu() - want).abs()[ok].max())
            assert int(ok.sum()) >= 0.25 * ok.numel() and err <= 1e-6, (tag, p, int(ok.sum()), err)
    get_context(DEV).sync_check()


# ------------------------------------------------------------------------------------------ fused maps, teacher-forced
# As test_gpu_region.test_fused_region_maps_teacher_forced: T is the fp16 restatement, E the fp64 network, both on the kernel's
# fp32 inputs at the kernel's own depths, composited in fp64 with the edits (appearance_oracle.render_on_depths).
FP16_TWIN_FRACTION = 0.3
FLOORS = {"rgb": 1e-2, "depth": 1e-1, "acc": 1e-2, "ins": 1e-2, "weights": 1.0}
_TF = {}


def _tf_setup(ins_num):
    if ins_num not in _TF:
        nc, nf, wc, wf = make_models(101, 202, ins_num, DEV)
        nets = {}
        for tag, w in (("coarse", wc), ("fine", wf)):
            p32 = {k: v.to(DEV) for k, v in O.to_torch(w).items()}
            p64 = {k: v.to(DEV) for k, v in O.to_torch(w, torch.float64).items()}
            nets[tag, "T"] = lambda x, p=p32: H.mlp_forward_f16(p, x.to(DEV)).cpu()
            nets[tag, "E"] = lambda x, p=p64: O.mlp_forward(p, x.to(DEV).double()).cpu()
        _TF[ins_num] = (nc, nf, nets, _floater_region(nf, ins_num))
    return _TF[ins_num]


def _edit(ins_num):
    """Tints on half the labels, density 0.5 on a third, 2.0 on another third.  (At ins_num 93 the fp16 kernel sets aside 19
    to 21 of the 513 rays whatever the scales, 20 with no appearance at all: the cap is a property of these rays.)"""
    colour = {k: OB.tint((0.2 + 0.6 * (k % 3) / 2, 0.9 - 0.3 * (k % 2), 0.4)) for k in range(0, ins_num + 1, 2)}
    density = {k: (0.5 if k % 3 == 0 else 2.0) for k in range(ins_num + 1) if k % 3 != 2}
    return OB.Appearance(ins_num, colour=colour, density=density)


@pytest.mark.parametrize("variant", ["alone", "keep", "region"])
@pytest.mark.parametrize("ins_num", [13, 93])
@pytest.mark.parametrize("impl", [pytest.param(_lib.IMPL_UMMA, id="exact"), pytest.param(_lib.IMPL_UMMA_F16, id="f16")])
def test_fused_appearance_maps_teacher_forced(impl, ins_num, variant):
    """The fused kernel with a tint and density-scale appearance (alone, with keep_objects, or with a floater region) on 513
    rays: every map and weight of both passes against E (exact: 1e-4 with a floor of a tenth of each map's scale) or within
    FP16_TWIN_FRACTION of T's distance to E (fp16, plus 4x the distance of an fp32 composite of T's own raw), on the kernel's
    own depths.  A ray is set aside only where a label that matters is ambiguous: at most 1 % of the rays exact, 4 % fp16."""
    from dmnerf_b200.autograd import mlp_forward_rays
    f16 = impl == _lib.IMPL_UMMA_F16
    nc, nf, nets, region = _tf_setup(ins_num)
    app = _edit(ins_num)
    keep_objects = [k for k in range(ins_num + 1) if k % 5 != 3] if variant == "keep" else None
    reg = region if variant == "region" else None
    wl, ro, rd = _rays("dmsr_study", 513)
    with torch.no_grad():
        got = render_rays(ro, rd, nc, nf, _z(wl), want_raw=False, want_samples=True, impl=impl, keep_objects=keep_objects,
                          region=reg, appearance=app)
        logits = {p: mlp_forward_rays(net, ro, rd, got["z_vals_" + p].contiguous(), impl).cpu().double()
                  for p, net in (("coarse", nc), ("fine", nf))}
    get_context(DEV).sync_check()
    keep = None
    if keep_objects is not None:
        keep = torch.zeros(ins_num + 1, dtype=torch.bool)
        keep[keep_objects] = True
    ex = None
    if reg is not None:
        ex = RO.exclusion(reg.voxel_map, reg.bits.cpu().numpy().view(np.uint32), reg.dim, reg.applies_words(ins_num),
                          reg.outside == "keep", ro.cpu().numpy(), rd.cpu().numpy())
    roc, rdc = ro.cpu(), rd.cpu()
    zs = {p: got["z_vals_" + p].cpu() for p in ("coarse", "fine")}
    refs = {r: AO.render_on_depths(nets["coarse", r], nets["fine", r], roc, rdc, zs["coarse"], zs["fine"], keep=keep, exclude=ex,
                                   appearance=app) for r in ("T", "E")}
    R = refs["T" if f16 else "E"]
    n = ro.shape[0]
    ambiguous = torch.zeros(n, dtype=torch.bool)
    for p in ("coarse", "fine"):
        lg = logits[p].reshape(R["raw_" + p].shape)
        diff = (torch.sigmoid(lg[..., 4:]) - torch.sigmoid(R["raw_" + p][..., 4:])).abs().amax(-1)
        trans = 1.0 - torch.cumsum(R["weights_" + p], -1) + R["weights_" + p]
        matters = (R["raw_" + p][..., 3] > 0) & (trans > 1e-6)
        ambiguous |= ((R["gap_" + p] < 4.0 * diff) & matters).any(-1)
    n_aside = int(ambiguous.sum())
    print("\n  appearance %s ins_num %d %s: %d rays set aside" % ("f16" if f16 else "exact", ins_num, variant, n_aside))
    assert n_aside <= (0.04 if f16 else 0.01) * n, n_aside
    ok = ~ambiguous
    for p in ("coarse", "fine"):
        if f16:
            T, E = refs["T"], refs["E"]
            raw32 = T["raw_" + p].float()
            sel32 = raw32 if keep is None else OO.select_objects(raw32, keep)
            if ex is not None:
                sel32 = RO.exclude_samples(sel32, ex(zs[p], T["labels_" + p]))
            t32 = dict(zip(("rgb", "weights", "depth", "ins", "acc"), AO.composite(raw32, sel32, zs[p].float(), rdc.float(), app)))
        for m in ("rgb", "depth", "acc", "ins", "weights"):
            k = "%s_%s" % (m, p)
            K = got[k].cpu().double()[ok]
            if f16:
                k_t, t_e = H.rel_l2(K, T[k][ok]), H.rel_l2(T[k][ok], E[k][ok])
                floor = H.rel_l2(t32[m].double()[ok], T[k][ok])
                print("    %-16s K-T %.2e  T-E %.2e  ratio %.3f" % (k, k_t, t_e, k_t / max(t_e, 1e-300)))
                assert k_t <= FP16_TWIN_FRACTION * t_e + 4.0 * floor, (k, k_t, t_e, floor)
            else:
                ref = R[k][ok].numpy()
                e = max_rel_err(K.numpy(), ref, max(FLOORS[m], 0.1 * float(np.abs(ref).max())))
                print("    %-16s max rel err %.2e" % (k, e))
                assert e <= 1e-4, (k, e)


# ------------------------------------------------------------------------------------------ rejections
def test_rejections_leave_the_next_render_unchanged():
    wl, ro, rd = _rays("dmsr_study", 64)
    nc, nf, _, _ = make_models(101, 202, 13, DEV)
    ctx = get_context(DEV)
    with torch.no_grad():
        before = render_rays(ro, rd, nc, nf, _z(wl), want_raw=False, want_samples=True)
    lib, st, n = ctx.lib, ctx.stream(), ro.shape[0]
    z, out = _z(wl), torch.empty(n, 3, device=DEV)
    io = _lib.RenderIO(rays_o=ro.data_ptr(), rays_d=rd.data_ptr(), z_coarse=z.data_ptr(), rgb_fine=out.data_ptr())

    def render(table, n_labels):
        rows = _lib.floats(table, table.size)
        edit = _lib.Edit(appearance=C.cast(rows, C.POINTER(C.c_float)), appearance_labels=n_labels)
        io.edit = C.pointer(edit)
        return lib.dmnerf_render_forward(ctx.handle, io, n, 64, 128, 0, 0, st)
    good = OB.Appearance(13).table
    # a table of 0 labels, label counts outside [2, 128], NaN and inf entries, a negative scale
    for n_labels in (0, 1, 129):
        big = np.tile(good[:1], (max(n_labels, 1), 1))
        assert render(big, n_labels) != 0
        assert b"labels outside" in lib.dmnerf_last_error()
    for i, v in ((3, float("nan")), (12, float("inf")), (14, float("nan"))):
        bad = good.copy()
        bad[5, i] = v
        assert render(bad, 14) != 0
        assert b"not finite" in lib.dmnerf_last_error()
    bad = good.copy()
    bad[2, 12] = -0.5
    assert render(bad, 14) != 0
    assert b"negative density scale" in lib.dmnerf_last_error()
    # a table of the wrong length for the bound networks
    short = OB.Appearance(12).table
    assert render(short, 13) != 0
    assert b"13 rows for 14 labels" in lib.dmnerf_last_error()
    with torch.no_grad(), pytest.raises(ValueError, match="ins_num 12"):
        render_rays(ro, rd, nc, nf, z, appearance=OB.Appearance(12))
    # grad mode
    with pytest.raises(RuntimeError, match="inference-only"):
        render_rays(ro, rd, nc, nf, z, appearance=OB.Appearance(13))
    with pytest.raises(RuntimeError, match="inference-only"):
        render_frame(48, 64, wl["K"], wl["c2w"], 4.0, 15.0, nc, nf, device=DEV, appearance=OB.Appearance(13))
    # nor does a render with an appearance leave anything behind: the next render without one is the unedited result
    with torch.no_grad():
        render_rays(ro, rd, nc, nf, z, want_raw=False, appearance=OB.Appearance(13, density={1: 0.5}))
        after = render_rays(ro, rd, nc, nf, _z(wl), want_raw=False, want_samples=True)
    _equal(before, after, before.keys())
    ctx.sync_check()


# ------------------------------------------------------------------------------------------ the tool
def test_render_objects_tool_appearance(tmp_path):
    nc, nf, _, _ = make_models(7, 8, 13, "cpu")
    ck = str(tmp_path / "ck.tar")
    torch.save({"network_coarse_state_dict": nc.state_dict(), "network_fine_state_dict": nf.state_dict()}, ck)
    wl = synth.workload("dmsr_study")
    Hh, W = 48, 64
    K = synth.dmsr_intrinsics(Hh, W)
    np.save(str(tmp_path / "pose.npy"), wl["c2w"])
    out = str(tmp_path / "out")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "render_objects.py"), ck, "--pose", str(tmp_path / "pose.npy"),
                        "--hwk", str(Hh), str(W)] + [repr(float(v)) for v in K.reshape(-1)] +
                       ["--tint", "1", "1", "0.2", "0.2", "--tint", "2", "1", "1", "1", "--opacity", "3", "0.3",
                        "--opacity", "4", "0", "--out", out],
                       capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["frames"] == 1 and sorted(os.listdir(out)) == ["000.png", "instance_000.png"]
