"""GPU: the training step's stage composite, emptiness penalizer and Hungarian instance loss against fp64, teacher-forced on the
kernels' own fp32 inputs (oracle/fp64_oracle.py, references run on the device).  Every discrete decision -- a sample's label, a
penalizer mask, the assignment -- is the fp32 rule's, so it is the kernel's; the arithmetic is held to 2x a first-order fp32
rounding budget computed from the same inputs (validated against the fp32 oracles in tests/test_fp64_budget_host.py), on every
element, at the sizes and head widths the kernels run.  Each case prints its worst error / budget ratio (pytest -s)."""
import numpy as np
import pytest
import torch
from scipy.optimize import linear_sum_assignment

from dmnerf_b200 import _lib, synth
from dmnerf_b200 import objects as OB
from dmnerf_b200.engine import get_context
from oracle import dmnerf_oracle as O
from oracle import fp64_oracle as F
from oracle import region_oracle as RO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MAPS = ("rgb", "weights", "depth", "ins", "acc")
SLACK = 2.0


def _i32(t):
    return _lib.ptr(t, torch.int32)


def _ratio(got, ref, budget):
    """Worst |got - ref| / budget over the elements (NaN anywhere, in the output or in the budget, fails)."""
    got, ref = got.to(ref.device).double(), ref.double()
    assert got.shape == ref.shape and bool(torch.isfinite(got).all()), (got.shape, ref.shape)
    assert bool(torch.isfinite(budget).all()) and bool(torch.isfinite(ref).all()), "budget or reference not finite"
    err = (got - ref).abs()
    return float(torch.where(err > 0, err / budget.to(ref.device), torch.zeros_like(err)).max()) if err.numel() else 0.0


def _check(what, ratios):
    print("\n  %s: error / budget %s" % (what, " ".join("%s %.3f" % kv for kv in ratios.items())))
    bad = {k: v for k, v in ratios.items() if not v <= SLACK}
    assert not bad, (what, bad)


# ------------------------------------------------------------------------------------------------------------ composite
def _composite_call(raw, z, rd, keep_all, keep_words=None, skip=None):
    """dmnerf_composite (raw ABI) -> dict of the five outputs; `skip` names one output passed as NULL."""
    n, s, c = raw.shape
    n_ins = c - 4 if keep_all else c - 5
    e = lambda *shape: torch.full(shape, float("nan"), device=DEV)
    out = {"rgb": e(n, 3), "weights": e(n, s), "depth": e(n), "ins": e(n, n_ins), "acc": e(n)}
    p = {k: (None if k == skip or v.numel() == 0 else _lib.ptr(v)) for k, v in out.items()}
    keep = None if keep_words is None else _lib.keep_mask(keep_words)
    get_context(DEV).call("dmnerf_composite", _lib.ptr(raw), _lib.ptr(z), _lib.ptr(rd), n, s, c, int(keep_all), keep, p["rgb"],
                          p["weights"], p["depth"], p["ins"], p["acc"])
    return out


def _n_rays(S, k):
    """The ray counts of a composite case: 1, 3, 4, 5 (a part of one 4-warp block) and 1023 (255 full blocks and a part),
    1023 rays also at S >= 3072 for the narrow heads; the widest heads there stop at 255 rays (a 1023 x 4096 x 132 case needs
    over 20 GB for its fp64 reference alone)."""
    return (1, 3, 4, 5, 1023 if S < 3072 or k <= 29 else 255)


def _composite_case(n, S, k, seed, keep_all):
    raw, z, rd = F.composite_inputs(n, S, k, seed, device=DEV)
    ratios = {}
    got = _composite_call(raw, z, rd, keep_all)
    ref = F.composite64(raw, z, rd, keep_all)
    budget = F.composite_budget(raw, z, rd, keep_all)
    assert not bool(ref["near"].any())
    for m in MAPS:
        ratios[m] = _ratio(got[m], ref[m], budget[m])
    for skip in MAPS:                                                  # each output NULL in turn: the others are unchanged
        part = _composite_call(raw, z, rd, keep_all, skip=skip)
        for m in MAPS:
            if m != skip:
                assert torch.equal(part[m], got[m]), (skip, m)
        assert bool(torch.isnan(part[skip]).all()), skip
    if k >= 2:                                                         # the select kernel, with exact ties split by the keep set
        keep = F.keep_split(k, seed).to(DEV)
        words = OB.object_mask(k - 1, keep=[i for i in range(k) if bool(keep[i])])
        got = _composite_call(raw, z, rd, keep_all, keep_words=words)
        ref = F.composite64(raw, z, rd, keep_all, keep=keep)
        budget = F.composite_budget(raw, z, rd, keep_all, keep=keep)
        for m in MAPS:
            ratios["keep_" + m] = _ratio(got[m], ref[m], budget[m])
    return ratios


@pytest.mark.parametrize("keep_all", [False, True])
@pytest.mark.parametrize("S,k", [(S, k) for S in (1, 2, 31, 32, 33, 64, 192, 1024, 3072, 3073, 4096) for k in (1, 29, 128)]
                         + [(S, k) for S in (64, 192) for k in (2, 28, 60, 61, 92, 93, 124, 125)])
def test_composite_fp64(S, k, keep_all):
    """dmnerf_composite against composite64 on every element of every ray: densities negative, zero, 1e4 and 1e-30, zero-width
    bins, rays_d = 0, logits up to +-80, exact ties of the winning logit; k = 1 with keep_all off gives an empty ins map; S >
    3072 takes the opt-in shared-memory path, k > 92 the 4th and 5th passes of the channel loop."""
    worst = {}
    for n in _n_rays(S, k):
        for key, v in _composite_case(n, S, k, seed=S * 1000 + k * 7 + n, keep_all=keep_all).items():
            worst[key] = float(np.maximum(worst.get(key, 0.0), v))           # NaN-propagating, unlike max()
    _check("composite S %d k %d keep_all %d" % (S, k, keep_all), worst)


@pytest.mark.parametrize("S,k", [(64, 14), (192, 14), (64, 94), (192, 94)])
def test_composite_fp64_training_sizes(S, k):
    """1024 rays of 64 coarse or 192 fine samples, at ins_num 13 and 93 (k = ins_num + 1)."""
    _check("composite 1024 x %d k %d" % (S, k), _composite_case(1024, S, k, seed=S + k, keep_all=False))


# ------------------------------------------------------------------------------------------------------------ stage render
def _half_region(ins_num, outside):
    """Half of a 32^3 grid over [-4, 4]^3 (the points with i < 16), applying to every label."""
    dim = 32
    vm = np.zeros((3, 4), dtype=np.float32)
    for a in range(3):
        vm[a, a], vm[a, 3] = (dim - 1) / 8.0, 4.0 * (dim - 1) / 8.0
    mask = np.zeros((dim, dim, dim), dtype=bool)
    mask[:dim // 2] = True
    bits = torch.from_numpy(RO.pack(mask).view(np.int32).copy()).to(DEV)
    return OB.Region(bits, dim, vm, outside=outside)


@pytest.mark.parametrize("edit", ["keep", "region_keep", "region_drop", "appearance"])
@pytest.mark.parametrize("name,ins_num", [("dmsr_study", 13), ("replica_room0_93", 93)])
@pytest.mark.parametrize("impl", [pytest.param(_lib.IMPL_UMMA, id="exact"), pytest.param(_lib.IMPL_UMMA_F16, id="f16")])
def test_stage_render_edit_teacher_forced(impl, name, ins_num, edit):
    """render_rays(want_raw=True) with an edit, each pass's maps against composite64 of the returned raw at the returned depths
    (labels from that raw: exact up to flagged near ties, which may be at most 0.1 % of the samples; only a ray on which a
    flagged sample carries weight is set aside)."""
    from dmnerf_b200.render import render_rays
    from dmnerf_b200.testing import make_models
    wl = synth.workload(name)
    sel = np.linspace(0, wl["H"] * wl["W"] - 1, 517).astype(np.int64)
    ro = torch.from_numpy(wl["rays_o"][sel]).to(DEV).contiguous()
    rd = torch.from_numpy(wl["rays_d"][sel]).to(DEV).contiguous()
    nc, nf, _, _ = make_models(101, 202, ins_num, DEV)
    kw, keep, exclude, app = {}, None, None, None
    if edit == "keep":
        kw["keep_objects"] = [i for i in range(ins_num + 1) if i % 3 != 1]
        keep = torch.zeros(ins_num + 1, dtype=torch.bool, device=DEV)
        keep[kw["keep_objects"]] = True
    elif edit.startswith("region"):
        reg = _half_region(ins_num, edit.split("_")[1])
        kw["region"] = reg
        exclude = RO.exclusion(reg.voxel_map, reg.bits.cpu().numpy().view(np.uint32), reg.dim, reg.applies_words(ins_num),
                               reg.outside == "keep", ro.cpu().numpy(), rd.cpu().numpy())
    else:
        app = OB.Appearance(ins_num, colour={i: OB.tint((0.9, 0.25, 0.1)) for i in range(0, ins_num + 1, 2)},
                            density={i: (0.0 if i % 3 == 0 else 2.5) for i in range(ins_num + 1) if i % 3 != 2})
        kw["appearance"] = app
    with torch.no_grad():
        out = render_rays(ro, rd, nc, nf, O.z_val_sample(1, wl["near"], wl["far"], 64)[0].to(DEV), impl=impl, **kw)
    get_context(DEV).sync_check()
    ratios, flagged, total = {}, 0, 0
    for p in ("coarse", "fine"):
        raw, z = out["raw_" + p], out["z_vals_" + p]
        ex = None if exclude is None else (lambda zz, lab: exclude(zz, lab).to(DEV))
        ref = F.composite64(raw, z, rd, False, keep, ex, app)
        budget = F.composite_budget(raw, z, rd, False, keep, ex, app)
        flagged += int(ref["near"].sum())
        total += ref["near"].numel()
        ok = ~(ref["near"] & ref["carries"]).any(-1)
        for m in MAPS:
            ratios["%s_%s" % (m, p)] = _ratio(out["%s_%s" % (m, p)][ok], ref[m][ok], budget[m][ok])
    print("\n  stage render %s %s: %d of %d samples near-tied" % (name, edit, flagged, total))
    assert flagged <= 1e-3 * total, (flagged, total)
    _check("stage render %s %s %s" % ("f16" if impl == _lib.IMPL_UMMA_F16 else "exact", name, edit), ratios)


# ------------------------------------------------------------------------------------------------------------ penalizer
def _pen_forward(raw, z, depth, rd, tol, w, lo=0, hi=None):
    """dmnerf_penalizer_forward on rays [lo, hi) -> (loss [1], head bytes)."""
    ctx = get_context(DEV)
    n, s, c = raw.shape
    hi = n if hi is None else hi
    u8 = torch.uint8
    part = torch.empty(int(ctx.lib.dmnerf_penalizer_partials_bytes(hi - lo, s, c)), device=DEV, dtype=u8)
    loss = torch.empty(1, device=DEV)
    ctx.call("dmnerf_penalizer_forward", _lib.ptr(raw[lo:hi]), _lib.ptr(z[lo:hi]), _lib.ptr(depth[lo:hi]), _lib.ptr(rd[lo:hi]), hi - lo,
             s, c, tol, w, _lib.ptr(part, u8), _lib.ptr(loss))
    return loss, part[:int(ctx.lib.dmnerf_penalizer_state_bytes())]


def _head(state):
    """(n_before, n_middle, sum_before, sum_middle) of a penalizer head."""
    h = state.cpu().numpy()
    return int(h[0:8].view(np.uint64)[0]), int(h[8:16].view(np.uint64)[0]), float(h[16:24].view(np.float64)[0]), \
        float(h[24:32].view(np.float64)[0])


def _pen_backward(raw, z, depth, rd, tol, w, state, g_loss, d_raw, accumulate, lo=0, hi=None):
    n, s, c = raw.shape
    hi = n if hi is None else hi
    get_context(DEV).call("dmnerf_penalizer_backward", _lib.ptr(raw[lo:hi]), _lib.ptr(z[lo:hi]), _lib.ptr(depth[lo:hi]),
                          _lib.ptr(rd[lo:hi]), hi - lo, s, c, tol, w, _lib.ptr(state, torch.uint8), _lib.ptr(g_loss),
                          _lib.ptr(d_raw[lo:hi]), int(accumulate))


@pytest.mark.parametrize("case", ["mixed", "before", "behind", "boundary", "zero_d", "saturated"])
@pytest.mark.parametrize("C", [5, 48, 49, 96, 97, 132])
@pytest.mark.parametrize("n,s", [(1, 1), (37, 64), (1024, 64), (1024, 192), (3072, 192), (300, 257)])
def test_penalizer_fp64(n, s, C, case):
    """Forward (loss and mask populations), backward at g_loss 1, 3 and 0, with and without accumulate (the preload's channels
    0..3 untouched), and the shards' partials and merge at world 1 to 3, against penalizer64 and its budget (2x)."""
    from dmnerf_b200.parallel import shard_range
    k = C - 4
    raw, z, depth, rd, tol, w = F.penalizer_inputs(n, s, k, seed=n * 3 + s + C, case="mixed" if case == "saturated" else case,
                                                   device=DEV)
    if case == "saturated":                                             # logits over +-16: p rounds to 0 or 1 in fp32
        raw = torch.where(raw >= 0, raw + 16.5, raw - 16.5)
    loss64, grad64, (before, middle) = F.penalizer64(raw, z, depth, rd, tol, w)
    d_loss, d_grad = F.penalizer_budget(raw, z, depth, rd, tol, w)
    loss, state = _pen_forward(raw, z, depth, rd, tol, w)
    nb, nm, _, _ = _head(state)
    assert (nb, nm) == (int(before.sum()), int(middle.sum()))
    ratios = {"loss": abs(float(loss) - float(loss64)) / d_loss if float(loss) != float(loss64) else 0.0}
    for world in (1, 2, 3):                                             # the shards' heads merged in rank order
        heads, pieces = [], [shard_range(n, world, r)[:2] for r in range(world)]
        for lo, hi in pieces:
            heads.append(_pen_forward(raw, z, depth, rd, tol, w, lo, hi)[1])
        merged, mloss = torch.empty_like(state), torch.empty(1, device=DEV)
        get_context(DEV).call("dmnerf_penalizer_merge", _lib.ptr(torch.stack(heads), torch.uint8), world, C,
                              _lib.ptr(merged, torch.uint8), _lib.ptr(mloss))
        assert _head(merged)[:2] == (nb, nm)
        if world == 1:                                                  # one shard: the single-process head and loss, bit for bit
            assert torch.equal(merged[:32], state[:32]) and torch.equal(mloss, loss)
        ratios["loss_w%d" % world] = abs(float(mloss) - float(loss64)) / d_loss if float(mloss) != float(loss64) else 0.0
        d_raw = torch.empty_like(raw)
        one = torch.ones(1, device=DEV)
        for lo, hi in pieces:
            _pen_backward(raw, z, depth, rd, tol, w, merged, one, d_raw, False, lo, hi)
        ratios["grad_w%d" % world] = _ratio(d_raw, grad64, d_grad)
    for g in (1.0, 3.0, 0.0):
        g_loss = torch.full((1,), g, device=DEV)
        d_raw = torch.full_like(raw, float("nan"))
        _pen_backward(raw, z, depth, rd, tol, w, state, g_loss, d_raw, False)
        assert bool((d_raw[..., :4] == 0).all())
        d_g = d_grad * g                                                # the gradient's budget is linear in g_loss
        ratios["grad_g%g" % g] = _ratio(d_raw, grad64 * g, d_g)
        pre = torch.randn(raw.shape, generator=torch.Generator(DEV).manual_seed(n + s), device=DEV)
        acc = pre.clone()
        _pen_backward(raw, z, depth, rd, tol, w, state, g_loss, acc, True)
        assert torch.equal(acc[..., :4], pre[..., :4])
        want = pre.double() + grad64 * g
        ratios["acc_g%g" % g] = _ratio(acc, want, d_g + F.U * want.abs())
    _check("penalizer %d x %d C %d %s" % (n, s, C, case), ratios)


@pytest.mark.parametrize("C", [5, 49, 97, 132])
@pytest.mark.parametrize("n,s", [(1024, 64), (1024, 192), (3072, 192)])
def test_penalizer_sums_exact(n, s, C):
    """rays_d = 0 puts every sample in the middle shell with the same gaussian, and logits of -20, 0 and 20 make its term one
    of three fp32 values on any implementation.  Their sum in fp64 is exact in any order (at most 2^20 terms of 24 bits within
    5 binades), so the head's middle sum and population and the loss are the exact ones, bit for bit."""
    gen = torch.Generator().manual_seed(n + s + C)
    raw = torch.randn(n, s, C, generator=gen)
    raw[..., -1] = (torch.randint(0, 3, (n, s), generator=gen).float() - 1.0) * 20.0
    raw, z = raw.to(DEV), (torch.rand(n, s, generator=gen).sort(-1).values * 11 + 4).to(DEV)
    depth, rd = (z[:, s // 2] + 0.01).contiguous(), torch.zeros(n, 3, device=DEV)
    tol, w = 0.05, 0.05
    # the kernel's fp32 steps on the device: g = expf(0) / (0.4 sqrt(2 pi)) + 1e-8, term = -logf(1 - p + 1e-8) g
    f = lambda v: torch.tensor(v, dtype=torch.float32, device=DEV)
    g = torch.exp(f(0.0)) / (f(0.4) * torch.sqrt(f(6.283185307179586))) + f(1e-8)
    p = torch.sigmoid(raw[..., -1])
    term = -torch.log((1.0 - p) + f(1e-8)) * g
    assert set(term.unique().tolist()) <= {0.0, float(-torch.log(f(0.5)) * g), float(-torch.log(f(1e-8)) * g)}
    exact = sum(float(v) * int((term == v).sum()) for v in term.unique())
    loss, state = _pen_forward(raw, z, depth, rd, tol, w)
    nb, nm, sb, sm = _head(state)
    assert (nb, nm, sb) == (0, n * s, 0.0)
    assert sm == exact, (sm, exact, (sm - exact) / exact)
    assert float(loss) == float(np.float32(exact / (n * s))), (float(loss), exact / (n * s))


# ------------------------------------------------------------------------------------------------------------ instance loss
def _ins_case(n, k, case, seed):
    from dmnerf_b200.evaluator import _costs
    from dmnerf_b200.parallel import shard_range
    ctx = get_context(DEV)
    pred, labels = F.ins_inputs(n, k, seed, case)
    if len(torch.unique(labels)) > k:
        return None
    pred, labels = pred.to(DEV), labels.to(DEV)
    gt_row = torch.empty(n, device=DEV, dtype=torch.int32)
    nv = torch.empty(1, device=DEV, dtype=torch.int32)
    ctx.call("dmnerf_ins_label_rows", _i32(labels), n, k, _i32(gt_row), _i32(nv))
    c = _costs(pred, gt_row)
    roc = torch.empty(k, device=DEV, dtype=torch.int32)
    l3 = torch.empty(3, device=DEV)
    ctx.call("dmnerf_hungarian_assign", _lib.ptr(c["cost_ce"]), _lib.ptr(c["cost_siou"]), _lib.ptr(c["col_sum"]), _i32(nv), n, k,
             _i32(roc), _lib.ptr(l3))
    g3 = torch.tensor([0.7, 1.3, 2.1], device=DEV)
    d = torch.full_like(pred, float("nan"))
    ctx.call("dmnerf_ins_loss_backward", _lib.ptr(pred), _i32(gt_row), n, n, k, _i32(roc), _i32(nv), _lib.ptr(c["tp"]),
             _lib.ptr(c["col_sum"]), _lib.ptr(c["row_count"]), _lib.ptr(g3), _lib.ptr(d))
    roc_h = roc.cpu().numpy()
    budget, ref = F.ins_loss_budget(pred, labels, k, roc_h, g3=tuple(g3.tolist()))
    V = ref["n_valid"]
    # label rows and populations exact
    assert torch.equal(gt_row.long(), ref["gt_row"]) and int(nv) == V
    assert torch.equal(c["row_count"].double(), ref["row_count"])
    # the assignment: scipy's on the kernel's fp32 costs; optimal on the fp64 costs to within k ulp of the largest cost
    sc32 = (c["cost_ce"] + c["cost_siou"])[:V].cpu().numpy()
    rows, cols = linear_sum_assignment(sc32)
    want = np.full(k, -1)
    want[cols] = rows
    assert (roc_h == want).all(), (roc_h, want)
    sc64 = (ref["cost_ce"] + ref["cost_siou"])[:V].cpu().numpy()
    r64, c64 = linear_sum_assignment(sc64)
    assert sc64[rows, cols].sum() - sc64[r64, c64].sum() <= k * 2.0 ** -23 * max(np.abs(sc64).max(), 1.0)
    if V == k:
        assert float(l3[1]) == 0.0 and float(ref["losses"][1]) == 0.0
    ratios = {key: _ratio(c[key], ref[key], budget[key]) for key in ("cost_ce", "cost_siou", "tp", "col_sum")}
    ratios["losses"] = _ratio(l3, ref["losses"], budget["losses"])
    ratios["d_pred"] = _ratio(d, ref["d_pred"], budget["d_pred"])
    # the sharded path: bitmaps, ranks, partials and merge, the loss backward per shard -- the same values
    for world in (2, 3):
        pieces = [shard_range(n, world, r)[:2] for r in range(world)]
        bitmaps = torch.stack([torch.empty(_lib.LABEL_WORDS, device=DEV, dtype=torch.int32) for _ in pieces])
        for r, (lo, hi) in enumerate(pieces):
            ctx.call("dmnerf_ins_label_bitmap", _i32(labels[lo:hi]), hi - lo, _i32(bitmaps[r]))
        parts = torch.empty(world, 3 * k * (k + 1), device=DEV, dtype=torch.float64)
        rows_w = []
        for r, (lo, hi) in enumerate(pieces):
            gr = torch.empty(hi - lo, device=DEV, dtype=torch.int32)
            nvw = torch.empty(1, device=DEV, dtype=torch.int32)
            ctx.call("dmnerf_ins_label_rows_merged", _i32(bitmaps), world, _i32(labels[lo:hi]), hi - lo, k, _i32(gr), _i32(nvw))
            assert int(nvw) == V
            ctx.call("dmnerf_hungarian_partials", _lib.ptr(pred[lo:hi]), _i32(gr), hi - lo, k, _lib.ptr(parts[r], torch.float64))
            rows_w.append(gr)
        assert torch.equal(torch.cat(rows_w), gt_row)
        e = lambda *s: torch.empty(s, device=DEV, dtype=torch.float32)
        cw = {"cost_ce": e(k, k), "cost_siou": e(k, k), "tp": e(k, k), "col_sum": e(k), "row_count": e(k)}
        ctx.call("dmnerf_hungarian_costs_merged", _lib.ptr(parts, torch.float64), world, n, k,
                 *[_lib.ptr(cw[key]) for key in ("cost_ce", "cost_siou", "tp", "col_sum", "row_count")])
        assert torch.equal(cw["row_count"], c["row_count"])
        for key in ("cost_ce", "cost_siou", "tp", "col_sum"):
            ratios["%s_w%d" % (key, world)] = _ratio(cw[key], ref[key], budget[key])
        dw = torch.full_like(pred, float("nan"))
        for (lo, hi), gr in zip(pieces, rows_w):
            ctx.call("dmnerf_ins_loss_backward", _lib.ptr(pred[lo:hi]), _i32(gr), hi - lo, n, k, _i32(roc), _i32(nv),
                     _lib.ptr(cw["tp"]), _lib.ptr(cw["col_sum"]), _lib.ptr(cw["row_count"]), _lib.ptr(g3), _lib.ptr(dw[lo:hi]))
        ratios["d_pred_w%d" % world] = _ratio(dw, ref["d_pred"], budget["d_pred"])
    ctx.sync_check()
    return ratios


@pytest.mark.parametrize("case", ["one", "k", "sparse", "runs", "exact", "mixed"])
@pytest.mark.parametrize("k", [1, 2, 13, 31, 32, 33, 93, 127, 128])
@pytest.mark.parametrize("n", [1, 31, 32, 33, 255, 256, 257, 1024, 3072])
def test_ins_loss_fp64(n, k, case):
    """Label rows, costs, tp, col_sum, the device assignment, the three losses and d_pred, and the sharded path at world 2
    and 3, against ins_loss64 given the kernel's assignment (budget 2x)."""
    ratios = _ins_case(n, k, case, seed=n * 131 + k)
    if ratios is None:
        pytest.skip("more distinct labels than channels")
    _check("ins loss n %d k %d %s" % (n, k, case), ratios)
