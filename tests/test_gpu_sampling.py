"""GPU: the three pieces of code that place the renderer's samples, against the oracle's sampler fed their own inputs.

  * dmnerf_stratify (prep_z_kernel): the stratified coarse depths of render.py:40-47, bit for bit against O.stratify;
  * dmnerf_hier_sample (hier_sample_kernel): mid-point bins, sample_pdf over weights[1:-1], sort(cat(...)) (render.py:66-70),
    used by training, by want_raw renders and by moved renders;
  * the fused render kernel's own sampler (64 + 128 without raw output: every frame of the benchmark).

Every fine-depth check is teacher-forced: O.hier_sample gets the exact coarse depths and weights the kernel sampled from, so a
flip across a pdf jump caused by different coarse weights cannot explain a miss.  A kernel's z_fine [n, S + I] passes when
  1. it is non-decreasing wherever it is finite;
  2. the coarse depths are in it bit for bit, as a multiset;
  3. the other I values match the oracle's sorted samples within 1e-5 + 1e-4 |ref|; a miss only in a ray where
     O.sample_pdf_explained flags a sample (the inverse CDF itself is ill-conditioned there), in at most 2 % of the rays
     unless the summation order alone causes it (below);
  4. where the test owns the output buffer, no slot keeps the sentinel it was filled with.
The library sums the CDF in one warp's order, the reference's CPU cumsum in fp64: the two differ in the last bits, and where
the inverse CDF is ill-conditioned that moves a sample -- at u = 1 with an empty last bin (every ray of a deterministic draw:
which side of 1 the last knot rounds to picks the bin), or in bins whose mass is near the 1e-5 guard (common in the rays of
trained-like scenes).  Such rays exceed 2 % on several inputs here.  So rule 3 has two parts: (3a) every ray equals
O.sample_pdf_warp, the reference's arithmetic with the library's summation order, bit for bit;
(3b) against the reference, every miss is explained, and the 2 % cap holds for the misses that 3a's restatement does not
reproduce.
Rays whose oracle row holds NaN (NaN weights) must equal that row: the finite values sorted, then the NaNs.

Paths: the merge path runs for u = None when both runs are sorted; random, explicit or knot u, unsorted depths and NaN samples
take the rank sort; S = 1024 (any I) needs more than 48 KB of shared memory per block.  Each check prints the rays with an
explained miss and the largest such miss (pytest -s)."""
import numpy as np
import pytest
import torch

from dmnerf_b200 import _lib, synth
from dmnerf_b200 import objects as OB
from dmnerf_b200.engine import get_context
from dmnerf_b200.testing import make_models
from oracle import dmnerf_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENTINEL = -7.25e37
MISS_RAYS = 0.02
ONE_MINUS = float(np.float32(1.0) - np.float32(2.0 ** -24))       # 0.99999994, the largest float below 1


def _ctx():
    return get_context(DEV)


def _stratify(z_in, stride, t_rand, n, s):
    out = torch.full((n, s), SENTINEL, device=DEV)
    _ctx().call("dmnerf_stratify", _lib.ptr(z_in, strided=True), stride, _lib.ptr(t_rand), n, s, _lib.ptr(out))
    _ctx().sync_check()
    return out.cpu()


def _hier(zc, wc, ni, u=None):
    """dmnerf_hier_sample on CPU or CUDA inputs, into a sentinel-filled buffer -> z_fine [n, S + I] on the host."""
    zc, wc = zc.to(DEV).float().contiguous(), wc.to(DEV).float().contiguous()
    u = None if u is None else u.to(DEV).float().contiguous()
    n, s = zc.shape
    out = torch.full((n, s + ni), SENTINEL, device=DEV)
    _ctx().call("dmnerf_hier_sample", _lib.ptr(zc), _lib.ptr(wc), _lib.ptr(u), n, s, ni, _lib.ptr(out))
    _ctx().sync_check()
    return out.cpu()


def check_fine(what, zf, zc, wc, ni, u=None, owned=True):
    """Rules 1-4 for the fine depths zf of coarse depths zc and weights wc (u: the uniforms, None for the deterministic
    linspace).  Returns (rays with an explained miss, largest explained miss)."""
    zf, zc, wc = zf.detach().cpu(), zc.detach().cpu().float(), wc.detach().cpu().float()
    u = None if u is None else u.detach().cpu().float()
    n, s = zc.shape
    assert zf.shape == (n, s + ni), (what, tuple(zf.shape))
    if owned:
        assert not bool((zf == SENTINEL).any()), (what, "slots never written", int((zf == SENTINEL).sum()))
    det = u is None
    ref = O.hier_sample(zc, wc, ni, det=det, u=u)
    odd = ~torch.isfinite(ref).all(-1)                           # NaN weights: finite values sorted, then the NaNs
    if odd.any():
        torch.testing.assert_close(zf[odd], ref[odd], rtol=0, atol=0, equal_nan=True, msg=lambda m: "%s: %s" % (what, m))
    ok = ~odd
    zf, zc, wc, ref = zf[ok], zc[ok], wc[ok], ref[ok]
    u = None if u is None else u[ok]
    m = zf.shape[0]
    if m == 0:
        return 0, 0.0
    assert bool(torch.isfinite(zf).all()), (what, "non-finite fine depths")
    assert bool((zf[:, 1:] >= zf[:, :-1]).all()), (what, "not sorted")                                     # 1
    sc = zc.sort(-1).values.contiguous()
    zf = zf.contiguous()
    count = lambda seq, v: torch.searchsorted(seq, v, right=True) - torch.searchsorted(seq, v, right=False)
    assert bool((count(zf, sc) >= count(sc, sc)).all()), (what, "a coarse depth is missing")                # 2
    first = torch.searchsorted(zf, zf, right=False)
    coarse = (torch.arange(s + ni)[None] - first) < count(sc, zf)           # the first copies of each coarse value
    assert bool((coarse.sum(-1) == s).all()), what
    got = zf[~coarse].reshape(m, ni)
    mids = 0.5 * (zc[:, 1:] + zc[:, :-1])
    s_ref = O.sample_pdf(mids, wc[:, 1:-1], ni, det=det, u=u)
    want = s_ref.sort(-1).values
    tol = 1e-5 + 1e-4 * want.abs()
    order = O.sample_pdf_warp(mids, wc[:, 1:-1], ni, det=det, u=u).sort(-1).values
    off = (got != order).any(-1)                                                                            # 3a
    assert not bool(off.any()), (what, "differs from the summation-order restatement", int(off.sum()),
                                 float((got - order).abs().max()))
    err = (got - want).abs()
    miss = (err > tol).any(-1)                                                                              # 3b
    by_order = miss & ((order - want).abs() > tol).any(-1)
    n_rows, n_order = int(miss.sum()), int(by_order.sum())
    worst = float(err[miss].max()) if n_rows else 0.0
    print("  %-52s %5d rays: %4d with an explained miss (%4d reproduced by the summation order), largest %.3g"
          % (what, m, n_rows, n_order, worst))
    assert n_rows - n_order <= max(1, int(MISS_RAYS * m)), (what, n_rows, n_order, m, worst)
    rows = torch.nonzero(miss).flatten()
    for k in range(0, len(rows), 64):                                                   # bounded memory at S = 1024
        r = rows[k:k + 64]
        flagged = O.sample_pdf_explained(mids[r], wc[r][:, 1:-1], ni, det, None if u is None else u[r],
                                         (1e-5 + 1e-4 * s_ref[r].abs()).numpy())
        assert flagged.any(-1).all(), (what, "unexplained misses", r[~torch.from_numpy(flagged.any(-1))][:4].tolist(), worst)
    return n_rows, worst


# ---------------------------------------------------------------------------------------------------- inputs
def _depths(kind, n, s, gen):
    row = torch.linspace(2.0, 13.0, s)
    if kind == "shared":
        return row.expand(n, s).contiguous()
    strat = O.stratify(row.expand(n, s), torch.rand(n, s, generator=gen))
    if kind == "stratified":
        return strat
    if kind == "repeated":                                     # every depth twice: zero-width bins
        rep = torch.linspace(2.0, 13.0, (s + 1) // 2).repeat_interleave(2)[:s]
        return (rep[None] + torch.rand(n, 1, generator=gen)).contiguous()
    assert kind == "unsorted"                                  # the reference sorts the concatenation, so these are valid
    return torch.gather(strat, 1, torch.argsort(torch.rand(n, s, generator=gen), -1))


def _weights(kind, n, s, gen):
    w = torch.zeros(n, s)
    even, odd = slice(0, None, 2), slice(1, None, 2)
    if kind == "random":
        w = torch.rand(n, s, generator=gen)
    elif kind == "sparse":                                     # 80 % zeros: the 1e-5 guards decide most bins
        w = torch.rand(n, s, generator=gen) * (torch.rand(n, s, generator=gen) >= 0.8)
    elif kind == "zero":                                       # uniform through the 1e-5 guard
        pass
    elif kind == "ends":                                       # all mass where [1:-1] drops it
        w[even, 0] = 1.0
        w[odd, -1] = 1.0
    elif kind == "one_hot":                                    # first and last interior bin
        w[even, 1] = 1.0
        w[odd, -2] = 1.0
    elif kind == "magnitudes":                                 # 1e-30 .. 1, and subnormals
        w = 10.0 ** (-30.0 * torch.rand(n, s, generator=gen))
        w.view(-1)[::17] = 1e-40
        w.view(-1)[5::23] = 1.4e-45
        w.view(-1)[9::29] = 0.0
    else:
        assert kind == "large"                                 # near 1e6: the total is ~6e7
        w = 1e6 * (1.0 + 0.01 * torch.rand(n, s, generator=gen))
    return w.float()


def _uniforms(n, ni, gen):
    """Random u with exact 0, 1 and 0.99999994 in every ray that has room for them."""
    u = torch.rand(n, ni, generator=gen)
    u[:, 0] = 0.0
    u[:, -1] = 1.0
    if ni > 2:
        u[:, ni // 2] = ONE_MINUS
    return u


def _u_cases(n, ni, gen):
    return (("u=None", None), ("u=random", _uniforms(n, ni, gen)), ("u=linspace", torch.linspace(0.0, 1.0, ni).expand(n, ni)))


def _run_u_cases(label, zc, wc, ni, gen):
    """dmnerf_hier_sample for u = None, random u and the explicit linspace, each checked by check_fine; the explicit linspace
    (rank sort) must equal u = None (merge path when both runs are sorted) bit for bit."""
    got = {}
    for tag, u in _u_cases(zc.shape[0], ni, gen):
        got[tag] = _hier(zc, wc, ni, u)
        check_fine("%s %s" % (label, tag), got[tag], zc, wc, ni, u)
    assert torch.equal(got["u=linspace"], got["u=None"]), label


# ------------------------------------------------------------------------------------------- A. stratified depths
@pytest.mark.parametrize("n", [1, 3, 257, 4097])
@pytest.mark.parametrize("s", [3, 4, 31, 32, 33, 64, 65, 1024])
def test_stratify_bit_exact(s, n):
    """dmnerf_stratify against O.stratify bit for bit (both are single-rounded fp32 operations in the same order): a shared row
    (stride 0), per-ray rows (stride S) and rows inside a wider tensor (stride S + 5, the extra columns hold values a read past
    the row would pick up); t_rand with exact 0, 0.99999994 and 1; without t_rand the rows come back unchanged."""
    gen = torch.Generator().manual_seed(1000 * s + n)
    row = torch.linspace(2.0, 13.0, s)
    per = (torch.rand(n, s, generator=gen) * 11.0 + 2.0).sort(-1).values
    wide = torch.rand(n, s + 5, generator=gen) * -99.0
    wide[:, :s] = per
    t = torch.rand(n, s, generator=gen)
    t.view(-1)[0::7] = 0.0
    t.view(-1)[1::7] = ONE_MINUS
    t.view(-1)[2::7] = 1.0
    wide_d = wide.to(DEV)
    for mode, z_in, stride, rows in (("shared", row.to(DEV), 0, row.expand(n, s)), ("per-ray", per.to(DEV), s, per),
                                      ("wide", wide_d[:, :s], s + 5, per)):
        assert torch.equal(_stratify(z_in, stride, None, n, s), rows.contiguous()), mode
        got = _stratify(z_in, stride, t.to(DEV), n, s)
        want = O.stratify(rows, t)
        assert torch.equal(got, want), (mode, int((got != want).sum()))


# -------------------------------------------------------------------------------- B. dmnerf_hier_sample, given inputs
SIZES_S = [3, 4, 33, 64, 65, 257, 1024]
SIZES_I = [2, 31, 32, 33, 128, 129, 2048]
N_RAYS = [1, 3, 4, 5, 1001]                    # 4 rays per block: 1, 3, 5 and 1001 leave the last block ragged


@pytest.mark.parametrize("ni", SIZES_I)
@pytest.mark.parametrize("s", SIZES_S)
def test_hier_sample_sizes(s, ni):
    """Every S x I of the supported range's edges on stratified depths and random weights (half of them zero), for u = None,
    random u and the explicit linspace.  The ray count cycles through N_RAYS; S = 1024 takes the large shared-memory launch."""
    n = N_RAYS[(SIZES_S.index(s) * len(SIZES_I) + SIZES_I.index(ni)) % len(N_RAYS)]
    if n == 1001 and s >= 257 and ni >= 2048:
        n = 5
    gen = torch.Generator().manual_seed(31 * s + ni)
    zc = _depths("stratified", n, s, gen)
    wc = torch.rand(n, s, generator=gen) * (torch.rand(n, s, generator=gen) < 0.5)
    _run_u_cases("S=%d I=%d n=%d" % (s, ni, n), zc, wc, ni, gen)


@pytest.mark.parametrize("depths", ["shared", "stratified", "repeated", "unsorted"])
@pytest.mark.parametrize("weights", ["random", "sparse", "zero", "ends", "one_hot", "magnitudes", "large"])
def test_hier_sample_weights_and_depths(weights, depths):
    """The production size (64 + 128) and a ragged one (65 + 129) on every kind of coarse weight and depth row, for u = None,
    random u and the explicit linspace."""
    for s, ni, n in ((64, 128, 1001), (65, 129, 5)):
        gen = torch.Generator().manual_seed(s + 7 * len(weights) + len(depths))
        _run_u_cases("S=%d I=%d %s/%s" % (s, ni, weights, depths), _depths(depths, n, s, gen), _weights(weights, n, s, gen), ni,
                     gen)


def _knot_case(n, s=66):
    """Coarse weights whose CDF is exact in any summation order: interior bins 0, 10, 11 and 40 hold 2^20 each (the 1e-5 guard
    rounds away), every other bin is empty (its mass, 1e-5 / 2^22, rounds away in every knot after the first).  The knots are 0,
    0.25 (bins 1-10), 0.5, 0.75 (bins 12-40) and 1 (bins 41-64), each shared by a run of empty bins."""
    gen = torch.Generator().manual_seed(66)
    zc = _depths("stratified", n, s, gen)
    wc = torch.zeros(n, s)
    wc[:, [1, 11, 12, 41]] = 2.0 ** 20
    return zc, wc


def test_hier_sample_u_on_cdf_knots():
    """u exactly at 0, 1 and on the CDF knots, where a run of empty bins follows the knot: searchsorted(right=True) takes the
    bin after the run, `>=` would take the one before it.  The CDF is exact, so nothing is ill-conditioned: the result equals
    O.hier_sample bit for bit, through the rank sort (explicit u) and through the merge path (u = None at I = 5 is the knots)."""
    n = 9
    zc, wc = _knot_case(n)
    knots = torch.tensor([0.0, 0.25, 0.5, 0.75, 1.0])
    u = knots[torch.arange(n * 32) % 5].reshape(n, 32)
    u = torch.gather(u, 1, torch.argsort(torch.rand(n, 32, generator=torch.Generator().manual_seed(5)), -1))
    for ni, uu in ((32, u), (5, None), (9, None)):
        got = _hier(zc, wc, ni, uu)
        want = O.hier_sample(zc, wc, ni, det=uu is None, u=uu)
        assert torch.equal(got, want), (ni, int((got != want).sum()))
        check_fine("knots I=%d %s" % (ni, "u" if uu is not None else "u=None"), got, zc, wc, ni, uu)


@pytest.mark.parametrize("det", [True, False], ids=["u=None", "u=random"])
def test_hier_sample_nan_weights(det):
    """NaN in one interior weight of one ray makes all of its importance samples NaN: that ray's row is the reference's (its
    coarse depths sorted, then the NaNs, which is torch.sort's order), every slot is written, and the other rays are what they
    are without the NaN.  A NaN in a weight that [1:-1] drops (w[:, 0], w[:, -1]) changes nothing."""
    n, s, ni = 7, 64, 128
    gen = torch.Generator().manual_seed(8)
    zc = _depths("stratified", n, s, gen)
    wc = _weights("random", n, s, gen)
    u = None if det else _uniforms(n, ni, gen)
    clean = _hier(zc, wc, ni, u)
    bad = wc.clone()
    bad[2, 17] = float("nan")
    bad[4, 0] = float("nan")
    bad[5, -1] = float("nan")
    got = _hier(zc, bad, ni, u)
    check_fine("NaN weights %s" % ("u=None" if det else "u=random"), got, zc, bad, ni, u)
    assert bool(torch.isnan(got[2, s:]).all()) and torch.equal(got[2, :s], zc[2].sort().values)
    keep = [r for r in range(n) if r != 2]
    assert torch.equal(got[keep], clean[keep])


@pytest.mark.parametrize("s,ni", [(2, 128), (1025, 128), (64, 1), (64, 2049)])
def test_hier_sample_size_limits(s, ni):
    """S outside [3, 1024] or I outside [2, 2048]: the call fails with a reported error, launches nothing, writes nothing."""
    n = 3
    zc, wc = torch.ones(n, s, device=DEV), torch.ones(n, s, device=DEV)
    out = torch.full((n, s + ni), SENTINEL, device=DEV)
    before = _lib.launch_count()
    with pytest.raises(RuntimeError, match="hier_sample"):
        _ctx().call("dmnerf_hier_sample", _lib.ptr(zc), _lib.ptr(wc), None, n, s, ni, _lib.ptr(out))
    assert _lib.launch_count() == before
    assert bool((out == SENTINEL).all())


# ------------------------------------------------------------------------------ C. the fused kernel's own sampler
_MODELS = {}


def _models(ins_num, shift=0.0):
    """(coarse, fine) networks of one head width; shift: added to the coarse density bias."""
    key = (ins_num, shift)
    if key not in _MODELS:
        nc, nf, _, _ = make_models(101, 202, ins_num, DEV)
        if shift:
            with torch.no_grad():
                dict(nc.named_parameters())["density_linear.bias"].add_(shift)
        _MODELS[key] = (nc.eval(), nf.eval())
    return _MODELS[key]


def _rays(name, n):
    wl = synth.workload(name)
    sel = np.linspace(0, wl["H"] * wl["W"] - 1, n).astype(np.int64)
    ro = torch.from_numpy(wl["rays_o"][sel]).to(DEV).contiguous()
    rd = torch.from_numpy(wl["rays_d"][sel]).to(DEV).contiguous()
    z = torch.linspace(0, 1, 64, device=DEV) * (wl["far"] - wl["near"]) + wl["near"]
    return wl, ro, rd, z


def _draws(n, perturb, seed):
    if not perturb:
        return {}
    gen = torch.Generator().manual_seed(seed)
    return dict(perturb=1.0, t_rand=torch.rand(n, 64, generator=gen).to(DEV), u=_uniforms(n, 128, gen).to(DEV))


def _check_render(what, out, z, kw, fused):
    """A render's coarse depths (the shared row, or O.stratify of it bit for bit) and its fine depths (rules 1-3 against
    O.hier_sample of its own coarse depths and weights).  The fused kernel's fine depths must also equal dmnerf_hier_sample's
    on the same two tensors bit for bit: both build the CDF with ray_build_cdf in one warp (same scan order), both sample with
    ray_sample_at and linspace01, and both sorts are exact."""
    zc, wc, zf = out["z_vals_coarse"].detach().cpu(), out["weights_coarse"].detach().cpu(), out["z_vals_fine"].detach().cpu()
    n = zc.shape[0]
    row = z.cpu().expand(n, 64)
    want = O.stratify(row, kw["t_rand"].cpu()) if "t_rand" in kw else row
    assert torch.equal(zc, want), (what, "coarse depths")
    u = kw.get("u")
    check_fine(what, zf, zc, wc, 128, u, owned=False)
    if fused:
        assert torch.equal(zf, _hier(zc, wc, 128, u)), (what, "fused and stage samplers differ")
    return wc


def _fused(what, ro, rd, nc, nf, z, kw, impl, **edit):
    from dmnerf_b200.render import render_rays
    ctx = _ctx()
    with torch.no_grad():
        ctx.bind(0, nc); ctx.bind(1, nf)
        first = render_rays(ro, rd, nc, nf, z, want_raw=False, want_samples=True, impl=impl, **kw, **edit)   # packs the images
        before = _lib.launch_count()
        out = render_rays(ro, rd, nc, nf, z, want_raw=False, want_samples=True, impl=impl, **kw, **edit)
        assert _lib.launch_count() - before == 1, (what, "not the fused kernel")
    ctx.sync_check()
    for k in ("z_vals_coarse", "weights_coarse", "z_vals_fine"):
        assert torch.equal(out[k], first[k]), (what, k)
    return _check_render(what, out, z, kw, fused=True)


IMPLS = [pytest.param(_lib.IMPL_UMMA, id="exact"), pytest.param(_lib.IMPL_UMMA_F16, id="f16")]


@pytest.mark.parametrize("n", [1, 257, 1001])
@pytest.mark.parametrize("perturb", [False, True], ids=["det", "perturb"])
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("name", ["dmsr_study", "replica_room0_93"])
def test_fused_sampler_teacher_forced(name, impl, perturb, n):
    """The fused 64 + 128 render's fine depths against O.hier_sample of its own coarse depths and weights, and against
    dmnerf_hier_sample on them bit for bit; odd ray counts leave the last ray pair half empty."""
    wl, ro, rd, z = _rays(name, n)
    nc, nf = _models(wl["ins_num"])
    _fused("%s %s n=%d" % (name, "perturb" if perturb else "det", n), ro, rd, nc, nf, z, _draws(n, perturb, n), impl)


def _region_box(ro, rd, wl, dim=16, half=False, outside="keep"):
    """A region over the box holding every sample point of the rays: the whole grid, or its lower half along the first axis."""
    pts = torch.cat([ro + rd * wl["near"], ro + rd * wl["far"]]).cpu().numpy()
    T, ext = OB.region_transform(pts.min(0) - 0.5, pts.max(0) + 0.5)
    mask = torch.ones((dim,) * 3, dtype=torch.bool, device=DEV)
    if half:
        mask[dim // 2:] = False
    return OB.region_from_mask(mask, T, ext, outside=outside)


@pytest.mark.parametrize("variant", ["keep_objects", "region", "appearance", "empty_selection", "empty_odd_rays",
                                     "density_shift"])
@pytest.mark.parametrize("impl", IMPLS)
def test_fused_sampler_edited_and_degenerate(variant, impl):
    """The selected fused kernels sample from edited weights: an object selection, a region covering half the grid, an
    appearance that scales densities.  Degenerate rays: an empty selection (every coarse weight zero), all-zero rays next to
    ordinary ones within one pair (odd rays moved outside a region that drops what lies outside it), and a coarse density
    bias of +1e6 that puts all the weight on the first sample, which [1:-1] drops.  Deterministic and perturbed."""
    if variant == "density_shift" and impl == _lib.IMPL_UMMA_F16:
        pytest.skip("the shifted density is checked on the exact network")
    n = 257
    wl, ro, rd, z = _rays("dmsr_study", n)
    ins_num = wl["ins_num"]
    nc, nf = _models(ins_num, 1e6 if variant == "density_shift" else 0.0)
    edit = {}
    if variant == "keep_objects":
        edit["keep_objects"] = [0, 2, 5, ins_num]
    elif variant == "region":
        edit["region"] = _region_box(ro, rd, wl, half=True)
    elif variant == "appearance":
        edit["appearance"] = OB.Appearance(ins_num, density={k: (0.0 if k % 3 == 0 else 2.5) for k in range(ins_num + 1)})
    elif variant == "empty_selection":
        edit["keep_objects"] = []
    elif variant == "empty_odd_rays":
        edit["region"] = _region_box(ro, rd, wl, outside="drop")
        ro = ro.clone()
        ro[1::2] += 1000.0
    for perturb in (False, True):
        what = "%s %s" % (variant, "perturb" if perturb else "det")
        wc = _fused(what, ro, rd, nc, nf, z, _draws(n, perturb, 3), impl, **edit)
        if variant == "empty_selection":
            assert float(wc.abs().max()) == 0.0
        elif variant == "empty_odd_rays":
            assert float(wc[1::2].abs().max()) == 0.0 and float((wc[0::2].sum(-1) > 0).float().mean()) > 0.9
        elif variant == "density_shift":
            assert float(wc[:, 0].min()) > 0.999 and float(wc[:, 1:-1].max()) < 1e-6


# ------------------------------------------------------------------------------------ D. training and stage paths
@pytest.mark.parametrize("name", ["dmsr_study", "replica_room0_93"])
def test_training_and_stage_samplers(name):
    """render_rays_grad (perturbed, given t_rand and u) and render_rays(want_raw=True), deterministic and perturbed: coarse depths
    O.stratify bit for bit, fine depths by rules 1-3 against O.hier_sample of the path's own coarse weights."""
    from dmnerf_b200.backward import render_rays_grad
    from dmnerf_b200.render import render_rays
    n = 1001
    wl, ro, rd, z = _rays(name, n)
    nc, nf, _, _ = make_models(101, 202, wl["ins_num"], DEV)
    kw = _draws(n, True, 21)
    out = render_rays_grad(ro, rd, nc, nf, z, N_importance=128, **kw)
    _check_render("%s training" % name, out, z, kw, fused=False)
    for perturb in (False, True):
        kw = _draws(n, perturb, 22)
        with torch.no_grad():
            out = render_rays(ro, rd, nc, nf, z, want_raw=True, **kw)
        _check_render("%s stage %s" % (name, "perturb" if perturb else "det"), out, z, kw, fused=False)
    _ctx().sync_check()
