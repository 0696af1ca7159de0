"""GPU: the fp16 preview network (IMPL_UMMA_F16) and the exact network (IMPL_UMMA) where kernels usually break -- every
object-head width the padded head stage distinguishes (ins_num 1, 13, 15, 16, 59, 93, 127: 16, 16, 16, 32, 64, 96, 128 head
rows), ragged batches whose tail tile is mostly padding rows, odd ray counts whose last ray pair is half empty, every ray in
either slot of its pair, the arg-max label walk of the selected kernels at 2 and 128 channels with exact ties, the stage path
(S != 64, N_importance != 128, want_raw) and host batches in parts.

References, all teacher-forced on the kernel's own depths:
  * T -- the fp16 restatement (oracle/dmnerf_f16.mlp_forward_f16), E -- the fp64 network, both on the kernels' fp32 inputs
    (dmnerf_f16.net_inputs_fp32: points, view directions and sin / cos formed in fp32 as the kernel forms them), so that the
    only difference between the fp16 kernel K and T is the fp32 accumulation order;
  * the composites of T and E run in fp64 (dmnerf_f16.render_on_depths).
The fp16 kernel must sit within FP16_TWIN_FRACTION of T's own distance to E (rel. L2, per map), FP16_GROUP_FRACTION per
channel group of the network output; a dropped or doubled pass, a wrong stage offset or a stale head row puts that ratio at 1
or above.  Where fp16 rounding does not move a
map at all (acc of rays that saturate), the kernel's fp32 composite is the only difference left, so the allowance adds 4x the
distance of an fp32 composite of T's own raw from T.  The exact network is held to 1e-4 against E.

The oracle networks run in fp64 on the device (dense GEMMs in double precision; where they run changes nothing but fp64
rounding), which keeps this file to a few minutes.  Every ratio is printed (pytest -s)."""
import numpy as np
import pytest
import torch

from dmnerf_b200 import _lib, synth
from dmnerf_b200.testing import make_models, max_rel_err, scale_err
from oracle import dmnerf_f16 as H
from oracle import dmnerf_oracle as O
from oracle import objects_oracle as OO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F16 = _lib.IMPL_UMMA_F16
NET_REL_L2 = 2e-3
FP16_TWIN_FRACTION = 0.3
# Per channel group of the network output the instance group sits higher (measured on an H100: 0.26 - 0.29 at ins_num >= 13,
# 0.34 - 0.35 at ins_num 1): its path has two more fp16 roundings (instance hidden layer, head), and every activation that the
# fp32 accumulation order pushes across an fp16 rounding boundary moves it by a whole fp16 ulp, a cascade that grows with the
# number of roundings; at 2 channels the group's own fp16 error against fp64 is the smallest.  A fault sits at 1 or above.
FP16_GROUP_FRACTION = 0.45
EXACT_TOL = 1e-4
IMPLS = [pytest.param(_lib.IMPL_UMMA, id="exact"), pytest.param(F16, id="f16")]
WIDTHS = [1, 13, 15, 16, 59, 93, 127]
GROUPS = (("rgb", slice(0, 3)), ("density", slice(3, 4)), ("ins", slice(4, None)))
# floors of the exact kernel's element-wise map comparison (test_baseline_config1_coarse_only_1024_rays); weights: absolute
FLOORS = {"rgb": 1e-2, "depth": 1e-1, "acc": 1e-2, "ins": 1e-2, "weights": 1.0}
MAPS = ("rgb", "depth", "acc", "ins", "weights")
WL = synth.workload("dmsr_study")

_MODELS = {}


def _models(ins_num):
    """(nc, nf, oracle networks) of one head width, built once per module: net[(pass, impl)] maps x [M, 90] -> raw (fp64)."""
    if ins_num not in _MODELS:
        nc, nf, wc, wf = make_models(101, 202, ins_num, DEV)
        _MODELS[ins_num] = (nc, nf, _oracle_nets(wc, wf))
    return _MODELS[ins_num]


def _oracle_nets(wc, wf):
    nets = {}
    for tag, w in (("coarse", wc), ("fine", wf)):
        p32, p64 = O.to_torch(w), O.to_torch(w, torch.float64)
        p32 = {k: v.to(DEV) for k, v in p32.items()}
        p64 = {k: v.to(DEV) for k, v in p64.items()}
        nets[tag, "T"] = lambda x, p=p32: H.mlp_forward_f16(p, x.to(DEV)).cpu()
        nets[tag, "E"] = lambda x, p=p64: O.mlp_forward(p, x.to(DEV).double()).cpu()
    return nets


def _rays(n, first=0):
    sel = np.linspace(first, WL["H"] * WL["W"] - 1, n).astype(np.int64)
    return torch.from_numpy(WL["rays_o"][sel]), torch.from_numpy(WL["rays_d"][sel])


def _sync():
    from dmnerf_b200.engine import get_context
    get_context(DEV).sync_check()


def _ratio_bound(what, k_t, t_e, floor=0.0, fraction=FP16_TWIN_FRACTION):
    """The fp16 kernel's distance to T against T's distance to E (+ the fp32 composite floor where given)."""
    ratio = k_t / max(t_e, 1e-300)
    print("    %-28s K-T %.2e  T-E %.2e  ratio %.3f%s" % (what, k_t, t_e, ratio, "" if not floor else "  (fp32 floor %.1e)" % floor))
    assert k_t <= fraction * t_e + 4.0 * floor, (what, k_t, t_e, ratio, floor)


# ============================================================================================ A. the network alone
def _network_case(mode):
    """(kernel call, twin inputs [M, 90] fp32, base rows, prefixes): mode x (embedded inputs), rays (S = 37) or points."""
    from dmnerf_b200.autograd import mlp_forward, mlp_forward_points, mlp_forward_rays
    n_rays, s = 56, 37                                  # 2072 rows; 37 is not a multiple of 32
    ro, rd = _rays(n_rays)
    gen = torch.Generator().manual_seed(5)
    z = (torch.rand(n_rays, s, generator=gen, dtype=torch.float64) * (WL["far"] - WL["near"]) + WL["near"]).float()
    pts = (ro[:, None, :] + rd[:, None, :] * z[..., None]).reshape(-1, 3)
    assert float(pts.abs().max()) < 64.0                 # the kernel's fast sin / cos in every warp: prefixes cannot flip it
    if mode == "rays":
        call = lambda net, impl, k: mlp_forward_rays(net, ro[:k].to(DEV), rd[:k].to(DEV), z[:k].to(DEV), impl).reshape(k * s, -1)
        return call, H.net_inputs_fp32(ro, rd, z), n_rays, [1, 3, 4, 7, 27, 55], s
    m = 2048
    dirs = (rd / torch.norm(rd, dim=-1, keepdim=True))[:, None, :].expand(n_rays, s, 3).reshape(-1, 3)
    pts, dirs = pts[:m].contiguous(), dirs[:m].contiguous()
    prefixes = [1, 2, 31, 127, 128, 129, 255, 257, 1000]
    if mode == "points":
        call = lambda net, impl, k: mlp_forward_points(net, pts[:k].to(DEV), dirs[:k].to(DEV), impl=impl)
        return call, H.points_inputs_fp32(pts, dirs), m, prefixes, 1
    x = H.net_inputs_fp32(ro, rd, z)[:m].contiguous()
    call = lambda net, impl, k: mlp_forward(net, x[:k].to(DEV), impl=impl)
    return call, x, m, prefixes, 1


@pytest.mark.parametrize("mode", ["x", "rays", "points"])
@pytest.mark.parametrize("ins_num", WIDTHS)
@pytest.mark.parametrize("impl", IMPLS)
def test_network_prefixes_and_accuracy(impl, ins_num, mode):
    """The fine network on ~2048 rows.  Every prefix of the batch gives the base call's first rows bit for bit (the padding rows
    of the tail tile contaminate nothing); on the base batch, per channel group: fp16 within FP16_TWIN_FRACTION of T's distance
    to E and within NET_REL_L2 of E; exact within 1e-4 of E (scale-relative)."""
    _, nf, nets = _models(ins_num)
    call, x_twin, base_n, prefixes, rows_per = _network_case(mode)
    with torch.no_grad():
        base = call(nf, impl, base_n)
        for k in prefixes:
            part = call(nf, impl, k)
            assert torch.equal(part, base[:k * rows_per]), (mode, k)
    _sync()
    got = base.cpu().double()
    ref64 = nets["fine", "E"](x_twin)
    assert got.shape == ref64.shape and torch.isfinite(got).all()
    print("\n  A %s ins_num %d %s:" % ("f16" if impl == F16 else "exact", ins_num, mode))
    if impl == F16:
        twin = nets["fine", "T"](x_twin)
        for g, sl in GROUPS:
            _ratio_bound(g, H.rel_l2(got[:, sl], twin[:, sl]), H.rel_l2(twin[:, sl], ref64[:, sl]), fraction=FP16_GROUP_FRACTION)
            assert H.rel_l2(got[:, sl], ref64[:, sl]) <= NET_REL_L2, (g, H.rel_l2(got[:, sl], ref64[:, sl]))
    else:
        for g, sl in GROUPS:
            e = scale_err(got[:, sl].numpy(), ref64[:, sl].numpy())
            print("    %-28s scale err %.2e" % (g, e))
            assert e <= EXACT_TOL, (g, e)


# ============================================================================================ B. the fused render
N_FUSED = 513


def _fused_inputs(case, n=N_FUSED):
    """rays, coarse depths (a shared [64] row, or per-ray rows when perturbed), kwargs of render_rays."""
    ro, rd = _rays(n)
    zrow = torch.linspace(WL["near"], WL["far"], 64)
    kw = {"keep_all_ins": case == "keep_all"}
    if case != "perturb":
        return ro, rd, zrow, kw
    gen = torch.Generator().manual_seed(17)
    z = zrow[None].expand(n, 64) + 0.02 * torch.rand(n, 1, generator=gen)
    kw.update(perturb=1.0, t_rand=torch.rand(n, 64, generator=gen), u=torch.rand(n, 128, generator=gen))
    return ro, rd, z.contiguous(), kw


def _render(nc, nf, ro, rd, z, kw, impl, keep_objects=None, rows=slice(None)):
    from dmnerf_b200.render import render_rays
    d = lambda t: t[rows].to(DEV)
    args = {k: (d(v) if torch.is_tensor(v) else v) for k, v in kw.items()}
    with torch.no_grad():
        return render_rays(d(ro), d(rd), nc, nf, z.to(DEV) if z.dim() == 1 else d(z), want_raw=False, want_samples=True,
                           impl=impl, keep_objects=keep_objects, **args)


def _teacher_forced(nets, ro, rd, out, keep=None, keep_all_ins=False):
    zc, zf = out["z_vals_coarse"].cpu(), out["z_vals_fine"].cpu()
    return {r: H.render_on_depths(nets["coarse", r], nets["fine", r], ro, rd, zc, zf, keep=keep, keep_all_ins=keep_all_ins)
            for r in ("T", "E")}


def _fp32_composite(ref, z, rd, p, keep=None, keep_all_ins=False):
    """The fp32 composite of a reference's own raw: what the kernel's fp32 composite alone does to that reference's maps."""
    raw = ref["raw_" + p] if keep is None else OO.select_objects(ref["raw_" + p], keep)
    return dict(zip(("rgb", "weights", "depth", "ins", "acc"),
                    O.composite(raw.float(), z.float(), rd.float(), keep_all_ins=keep_all_ins)))


def _check_maps(impl, got, refs, rd, rays, label, keep=None, keep_all_ins=False, scale_floor=False):
    """fp16: rel_l2(K, T) <= FP16_TWIN_FRACTION rel_l2(T, E) (+ the fp32 composite floor) for every coarse and fine map;
    exact: max_rel_err(K, E) <= 1e-4 with FLOORS, or with scale_floor at least a tenth of the map's largest value (the
    convention of testing.error_stats).  Over the rays `rays` (a bool mask)."""
    print("\n  %s:" % label)
    T, E = refs["T"], refs["E"]
    for p in ("coarse", "fine"):
        t32 = _fp32_composite(T, got["z_vals_" + p].cpu(), rd, p, keep, keep_all_ins) if impl == F16 else None
        for m in MAPS:
            k = "%s_%s" % (m, p)
            K = got[k].cpu().double()[rays]
            if impl == F16:
                tm, em = T[k][rays], E[k][rays]
                _ratio_bound(k, H.rel_l2(K, tm), H.rel_l2(tm, em), H.rel_l2(t32[m].double()[rays], tm))
            else:
                ref = E[k][rays].numpy()
                floor = max(FLOORS[m], 0.1 * float(np.abs(ref).max())) if scale_floor else FLOORS[m]
                e = max_rel_err(K.numpy(), ref, floor)
                i = np.unravel_index(np.argmax(np.abs(K.numpy() - ref) / np.maximum(np.abs(ref), floor)), ref.shape)
                print("    %-28s max rel err %.2e  (at %s: %.6e vs fp64 %.6e)" % (k, e, i, float(K.numpy()[i]), float(ref[i])))
                assert e <= EXACT_TOL, (k, e)


def _check_depths(got, z, kw):
    """Coarse depths: the shared row or the fp32 stratification, bit for bit.  Fine depths: sort(cat(zc, sample_pdf in fp32 of
    the kernel's own coarse weights)), every miss one that sample_pdf itself makes ill-conditioned."""
    n = got["z_vals_coarse"].shape[0]
    zc = got["z_vals_coarse"].cpu()
    want = O.stratify(z.float(), kw["t_rand"].float()) if "t_rand" in kw else z.float()[None].expand(n, 64)
    assert torch.equal(zc, want)
    wc = got["weights_coarse"].cpu()
    mids = 0.5 * (zc[:, 1:] + zc[:, :-1])
    det, u = "u" not in kw, kw.get("u")
    s_ref = O.sample_pdf(mids, wc[:, 1:-1], 128, det=det, u=u)
    zf = got["z_vals_fine"].cpu()
    tol = 1e-5 + 1e-4 * s_ref.abs()
    idx = torch.searchsorted(zf.contiguous(), s_ref.contiguous()).clamp(max=zf.shape[1] - 1)
    near = torch.minimum((torch.gather(zf, 1, idx) - s_ref).abs(), (torch.gather(zf, 1, (idx - 1).clamp(min=0)) - s_ref).abs())
    miss = (near > tol).numpy()
    if miss.any():
        unexplained = miss & ~O.sample_pdf_explained(mids, wc[:, 1:-1], 128, det, u, tol.numpy())
        assert not unexplained.any(), (int(unexplained.sum()), int(miss.sum()))
    clean = ~torch.from_numpy(miss.any(-1))
    z_ref = torch.sort(torch.cat([zc, s_ref], -1), -1).values
    assert bool(((zf - z_ref).abs() <= 1e-5 + 1e-4 * z_ref.abs())[clean].all())
    return int((~clean).sum())


@pytest.mark.parametrize("case", ["shared", "perturb", "keep_all"])
@pytest.mark.parametrize("ins_num", WIDTHS)
@pytest.mark.parametrize("impl", IMPLS)
def test_fused_render_edges_and_teacher_forced_maps(impl, ins_num, case):
    """render_rays on 513 rays (the last pair half empty): prefixes of 1, 2, 3 and 257 rays and the shift by one ray (every
    ray in the other slot of its pair) give the base call's rays bit for bit; coarse and fine depths as in _check_depths; every
    map and weight of both passes, over all rays, against T and E on the kernel's own depths (_check_maps)."""
    nc, nf, nets = _models(ins_num)
    ro, rd, z, kw = _fused_inputs(case)
    base = _render(nc, nf, ro, rd, z, kw, impl)
    for rows in (slice(0, 1), slice(0, 2), slice(0, 3), slice(0, 257), slice(1, None)):
        part = _render(nc, nf, ro, rd, z, kw, impl, rows=rows)
        for k, v in part.items():
            assert torch.equal(v, base[k][rows]), (rows, k)
    _sync()
    assert all(torch.isfinite(v).all() for v in base.values())
    flips = _check_depths(base, z, kw)
    refs = _teacher_forced(nets, ro, rd, base, keep_all_ins=kw["keep_all_ins"])
    label = "B %s ins_num %d %s (%d rays with a fine sample across a pdf jump)" % (
        "f16" if impl == F16 else "exact", ins_num, case, flips)
    _check_maps(impl, base, refs, rd, torch.ones(N_FUSED, dtype=torch.bool), label, keep_all_ins=kw["keep_all_ins"])


# ============================================================================================ C. object selection
@pytest.mark.parametrize("sel", ["keep", "remove"])
@pytest.mark.parametrize("ins_num", [1, 13, 127])
@pytest.mark.parametrize("impl", IMPLS)
def test_selected_render_teacher_forced(impl, ins_num, sel):
    """Keep {k} / remove {k} (k: the label most rays see) through the selected fused kernel, against T (fp16) or E (exact) with
    objects_oracle.select_objects on the kernel's own depths.  A ray is set aside only when one of its samples is ambiguous:
    the reference's two largest instance sigmoids closer than 4x the largest sigmoid difference between the kernel's logits
    (mlp_forward_rays at the same depths) and the reference's, at a sample whose label can change the maps (density > 0 and
    transmittance > 1e-6 in the reference).  At most 1 % of the rays may be for the exact network (measured on an H100:
    0.2 - 0.6 %), 4 % for fp16, whose sigmoid differences are ~100x larger (measured: 1.2 - 2.7 % at ins_num 13 and 127, none
    at 1; the renders are bit-reproducible, so the count is a property of these inputs).  The exact network's maps use a floor
    of a tenth of each map's scale: a selection leaves rays that only graze the kept object (acc 0.01 - 0.04), whose maps carry
    the relative error of a few small weights, i.e. of a density error bounded relative to the batch's largest density
    (measured: up to 1.6e-4 against the fixed floors, depth 0.1 - 0.2 on those rays)."""
    from dmnerf_b200.autograd import mlp_forward_rays
    nc, nf, nets = _models(ins_num)
    ro, rd, z, kw = _fused_inputs("shared")
    plain = _render(nc, nf, ro, rd, z, kw, impl)
    k_obj = int(torch.mode(plain["ins_fine"].argmax(-1).cpu()).values)               # the object most rays see
    keep = torch.zeros(ins_num + 1, dtype=torch.bool)
    keep[k_obj] = True
    if sel == "remove":
        keep = ~keep
    got = _render(nc, nf, ro, rd, z, kw, impl, keep_objects=keep.nonzero().flatten().tolist())
    with torch.no_grad():
        logits = {p: mlp_forward_rays(net, ro.to(DEV), rd.to(DEV), got["z_vals_" + p], impl).cpu().double()
                  for p, net in (("coarse", nc), ("fine", nf))}
    _sync()
    refs = _teacher_forced(nets, ro, rd, got, keep=keep)
    R = refs["T" if impl == F16 else "E"]
    ambiguous = torch.zeros(N_FUSED, dtype=torch.bool)
    for p in ("coarse", "fine"):
        diff = (torch.sigmoid(logits[p][..., 4:]) - torch.sigmoid(R["raw_" + p][..., 4:])).abs().amax(-1)
        # a label decides nothing where the sample's alpha is 0 either way (density <= 0) or no transmittance reaches it
        trans = 1.0 - torch.cumsum(R["weights_" + p], -1) + R["weights_" + p]
        matters = (R["raw_" + p][..., 3] > 0) & (trans > 1e-6)
        ambiguous |= ((R["gap_" + p] < 4.0 * diff) & matters).any(-1)
    n_aside = int(ambiguous.sum())
    assert n_aside <= (0.04 if impl == F16 else 0.01) * N_FUSED, n_aside
    label = "C %s ins_num %d %s {%d} (%d rays set aside)" % ("f16" if impl == F16 else "exact", ins_num, sel, k_obj, n_aside)
    _check_maps(impl, got, refs, rd, ~ambiguous, label, keep=keep, scale_floor=True)


@pytest.mark.parametrize("ins_num,a", [(1, 0), (127, 126)])
@pytest.mark.parametrize("impl", IMPLS)
def test_tied_labels_resolve_to_the_first(impl, ins_num, a):
    """ins_linear's row and bias of channel a copied into channel b = a + 1 in both networks, every channel below a lowered by
    30 (so a and b hold the largest logit of every sample): every sample ties exactly, so its
    label is a (first maximum, whichever channel a lane's walk starts at; (126, 127) is the end of the 128-channel walk).
    Keeping {b} alone leaves nothing (rgb = depth = acc = 0, ins = sigmoid(0) = 0.5); keeping {a} is keeping {a, b}."""
    from dmnerf_b200.autograd import mlp_forward_rays
    nc, nf, _, _ = make_models(101, 202, ins_num, DEV)
    b = a + 1
    with torch.no_grad():
        for net in (nc, nf):
            net.ins_linear.bias[:a] -= 30.0                          # every other channel far below a and b
            net.ins_linear.weight[b] = net.ins_linear.weight[a]
            net.ins_linear.bias[b] = net.ins_linear.bias[a]
    ro, rd, z, kw = _fused_inputs("shared", 257)
    only_b = _render(nc, nf, ro, rd, z, kw, impl, keep_objects=[b])
    only_a = _render(nc, nf, ro, rd, z, kw, impl, keep_objects=[a])
    both = _render(nc, nf, ro, rd, z, kw, impl, keep_objects=[a, b])
    with torch.no_grad():
        raw = mlp_forward_rays(nf, ro.to(DEV), rd.to(DEV), only_a["z_vals_fine"], impl)
    _sync()
    assert torch.equal(raw[..., 4 + a], raw[..., 4 + b])           # the tie is exact in the kernel's arithmetic
    for p in ("coarse", "fine"):
        for m in ("rgb", "depth", "acc"):
            assert not bool(only_b["%s_%s" % (m, p)].any()), (m, p)
        assert bool((only_b["ins_" + p] == 0.5).all()), p
        assert bool(only_a["acc_" + p].any()), p
    for k, v in only_a.items():
        assert torch.equal(v, both[k]), k


# ============================================================================================ D. the stage path
@pytest.mark.parametrize("case", ["48+64", "raw"])
@pytest.mark.parametrize("ins_num", WIDTHS)
@pytest.mark.parametrize("impl", IMPLS)
def test_stage_path_raw_and_maps(impl, ins_num, case):
    """render_rays on the stage-by-stage path (S = 48 with N_importance = 64, or want_raw=True at 64 + 128) on 257 rays:
    raw_coarse / raw_fine against T and E at the depths the call returns (fp16: the ratio and NET_REL_L2 bounds of A; exact:
    1e-4), and every map equal to the fp64 composite of the kernel's own raw to 1e-4."""
    from dmnerf_b200.render import render_rays
    nc, nf, nets = _models(ins_num)
    ro, rd = _rays(257)
    S, NI = (48, 64) if case == "48+64" else (64, 128)
    z = torch.linspace(WL["near"], WL["far"], S)
    with torch.no_grad():
        out = render_rays(ro.to(DEV), rd.to(DEV), nc, nf, z.to(DEV), N_importance=NI, want_raw=True, impl=impl)
    _sync()
    print("\n  D %s ins_num %d %s:" % ("f16" if impl == F16 else "exact", ins_num, case))
    for p in ("coarse", "fine"):
        zp = out["z_vals_" + p].cpu()
        got = out["raw_" + p].cpu().double().reshape(-1, 5 + ins_num)
        x = H.net_inputs_fp32(ro, rd, zp)
        ref64 = nets[p, "E"](x)
        if impl == F16:
            twin = nets[p, "T"](x)
            for g, sl in GROUPS:
                _ratio_bound("raw_%s %s" % (p, g), H.rel_l2(got[:, sl], twin[:, sl]), H.rel_l2(twin[:, sl], ref64[:, sl]),
                             fraction=FP16_GROUP_FRACTION)
                assert H.rel_l2(got[:, sl], ref64[:, sl]) <= NET_REL_L2
        else:
            for g, sl in GROUPS:
                e = scale_err(got[:, sl].numpy(), ref64[:, sl].numpy())
                print("    raw_%-24s scale err %.2e" % ("%s %s" % (p, g), e))
                assert e <= EXACT_TOL, (p, g, e)
        maps = O.composite(got.reshape(257, zp.shape[1], -1), zp.double(), rd.double())
        for m, ref in zip(("rgb", "weights", "depth", "ins", "acc"), maps):
            k = "%s_%s" % (m, p)
            e = max_rel_err(out[k].cpu().numpy(), ref.numpy(), FLOORS[m])
            assert e <= EXACT_TOL, (k, e)


# ============================================================================================ E. host batches
@pytest.mark.parametrize("impl", IMPLS)
def test_frame_pixel_ranges_are_slices_of_the_frame(impl):
    """render_frame of a 480 x 320 frame (153 600 rays: rendered in parts) and of pixel ranges with odd starts: the ranges are
    the matching slices of the whole frame, bit for bit."""
    from dmnerf_b200.render import render_frame
    nc, nf, _ = _models(13)
    H_, W_ = 480, 320
    K = synth.dmsr_intrinsics(H_, W_)
    with torch.no_grad():
        full = render_frame(H_, W_, K, WL["c2w"], WL["near"], WL["far"], nc, nf, impl=impl, device=DEV)
        full = {k: v.reshape(H_ * W_, -1) for k, v in full.items()}
        for begin, count in ((37, 101), (65537, 4097), (131071, 3)):
            part = render_frame(H_, W_, K, WL["c2w"], WL["near"], WL["far"], nc, nf, impl=impl, device=DEV,
                                pixel_range=(begin, count))
            for k, v in part.items():
                assert torch.equal(v.reshape(count, -1), full[k][begin:begin + count]), (begin, k)
    _sync()
    assert all(torch.isfinite(v).all() for v in full.values())
