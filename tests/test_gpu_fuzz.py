"""GPU: randomised differential tests (hypothesis) of the per-ray stage kernels against the oracle at ragged sizes -- ray counts
that are not multiples of a warp or a tile, sample counts from 3 to a few hundred, degenerate weights -- and of the domain's
size-independent properties (SURVEY.md 8c: sum of weights <= 1, merged depths sorted and within range, deterministic sampling
monotone, instance map in (0,1))."""
import numpy as np
import pytest
import torch
from hypothesis import given, settings, strategies as st, HealthCheck

pytestmark = pytest.mark.gpu

from dmnerf_b200.testing import max_rel_err, frac_bad
from oracle import dmnerf_oracle as O

DEV = "cuda"
COMMON = dict(max_examples=20, deadline=None, suppress_health_check=list(HealthCheck), derandomize=True)


def _cu(t):
    return t.to(DEV).contiguous()


@settings(**COMMON)
@given(n=st.integers(1, 70), s=st.integers(3, 260), k=st.integers(2, 40), seed=st.integers(0, 2 ** 20), keep=st.booleans())
def test_composite_fuzz(n, s, k, seed, keep):
    from dmnerf_b200.render import composite
    gen = torch.Generator().manual_seed(seed)
    raw = torch.randn(n, s, 4 + k, generator=gen) * 2
    raw[..., 3] = raw[..., 3] * 3 - 1                                       # plenty of negative (clamped) and large densities
    z = (torch.rand(n, s, generator=gen).sort(-1).values * 9 + 1)
    rd = torch.randn(n, 3, generator=gen) * 1.5
    ref = O.composite(raw, z, rd, keep_all_ins=keep)
    with torch.no_grad():
        got = composite(_cu(raw), _cu(z), _cu(rd), keep_all_ins=keep)
    rgb, w, depth, ins, acc = [g.cpu() for g in got]
    assert max_rel_err(w, ref[1], 1e-3) <= 1e-4 and max_rel_err(rgb, ref[0], 1e-2) <= 1e-4
    assert max_rel_err(depth, ref[2], 1e-1) <= 1e-4 and max_rel_err(ins, ref[3], 1e-2) <= 1e-4
    assert float(acc.max()) <= 1.0 + 1e-5 and float(w.min()) >= 0.0                       # transmittance is a probability
    assert ins.shape[1] == (k if keep else k - 1) and float(ins.min()) > 0.0 and float(ins.max()) < 1.0 + 1e-7


@settings(**COMMON)
@given(n=st.integers(1, 70), nb=st.integers(3, 130), ns=st.integers(2, 200), seed=st.integers(0, 2 ** 20), det=st.booleans(),
       sparse=st.booleans())
def test_sample_pdf_fuzz(n, nb, ns, seed, det, sparse):
    from dmnerf_b200.helpers import sample_pdf
    gen = torch.Generator().manual_seed(seed)
    bins = (torch.rand(n, nb, generator=gen).sort(-1).values * 10 + 2)
    w = torch.rand(n, nb - 1, generator=gen)
    if sparse:
        w = w * (torch.rand(n, nb - 1, generator=gen) < 0.2)                 # many empty bins: the 1e-5 guards matter
    u = None if det else torch.rand(n, ns, generator=gen)
    ref = O.sample_pdf(bins, w, ns, det=det, u=u).numpy()
    got = sample_pdf(_cu(bins), _cu(w), ns, det=det, u=None if u is None else _cu(u)).cpu().numpy()
    assert got.shape == ref.shape and np.isfinite(got).all()
    tol = 1e-5 + 1e-4 * np.abs(ref)
    bad = np.abs(got - ref) > tol
    assert bad.sum() <= max(2, 2e-2 * bad.size), (int(bad.sum()), bad.size)      # a tiny draw may have one or two ill-conditioned samples
    if bad.any():
        # every miss must be one the inverse CDF itself makes ill-conditioned, not an arithmetic error of the kernel
        unexplained = bad & ~O.sample_pdf_explained(bins, w, ns, det, u, tol)
        assert not unexplained.any(), (int(unexplained.sum()), int(bad.sum()), got[unexplained][:4], ref[unexplained][:4])
    assert got.min() >= float(bins.min()) - 1e-4 and got.max() <= float(bins.max()) + 1e-4
    if det:
        assert (np.diff(got, axis=-1) >= -1e-6).all()


@settings(**COMMON)
@given(n=st.integers(1, 70), na=st.integers(1, 130), nb=st.integers(1, 200), seed=st.integers(0, 2 ** 20), sort_b=st.booleans())
def test_sort_concat_fuzz(n, na, nb, seed, sort_b):
    from dmnerf_b200.helpers import sort_concat
    gen = torch.Generator().manual_seed(seed)
    a = (torch.rand(n, na, generator=gen) * 8).sort(-1).values
    b = torch.rand(n, nb, generator=gen) * 8
    b = b.sort(-1).values if sort_b else b
    t = min(na, nb, 3)
    b[:, :t] = a[:, :t]                                                    # ties between the two runs
    ref = torch.sort(torch.cat([a, b], -1), -1).values
    got = sort_concat(_cu(a), _cu(b)).cpu()
    assert torch.equal(got, ref)


@settings(**COMMON)
@given(m=st.integers(1, 300), seed=st.integers(0, 2 ** 20), scale=st.sampled_from([0.01, 1.0, 20.0]))
def test_posenc_fuzz(m, seed, scale):
    from dmnerf_b200.embedder import get_embedder
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(m, 3, generator=gen) * scale
    pe, ve = get_embedder(10)[0], get_embedder(4)[0]
    assert max_rel_err(pe.embed(_cu(x)).cpu(), O.embed(x, 10), 1e-2) <= 1e-4
    assert max_rel_err(ve.embed(_cu(x)).cpu(), O.embed(x, 4), 1e-2) <= 1e-4


@settings(max_examples=8, deadline=None, suppress_health_check=list(HealthCheck), derandomize=True)
@given(m=st.sampled_from([1, 2, 31, 127, 128, 129, 255, 257, 640, 1000]), ins_num=st.sampled_from([1, 13, 59, 127]),
       seed=st.integers(0, 2 ** 10))
def test_network_kernels_ragged_batches(m, ins_num, seed):
    """DM_NeRF.forward on the tensor-core kernel (and the fp32 kernel) for batch sizes around the 128-row tile and the
    extremes of the object-head width, against the oracle; the fp16 preview network against the fp64 oracle, rel. L2 over the
    whole output within the fp64 bound of tests/test_gpu_precision.py."""
    from dmnerf_b200 import synth, _lib
    from dmnerf_b200.testing import model_from_weights, scale_err, rel_l2
    w = synth.make_weights(500 + seed % 7, ins_num)
    net = model_from_weights(w, DEV).eval()
    gen = torch.Generator().manual_seed(seed)
    pts = torch.rand(m, 3, generator=gen) * 6 - 3
    vd = torch.randn(m, 3, generator=gen)
    vd = vd / vd.norm(dim=-1, keepdim=True)
    x = torch.cat([O.embed(pts, 10), O.embed(vd, 4)], -1)
    ref = O.mlp_forward(O.to_torch(w), x).numpy()
    with torch.no_grad():
        for impl, tol in ((_lib.IMPL_UMMA, 1e-4), (_lib.IMPL_SIMT, 2e-5)):
            got = net(_cu(x), impl=impl).cpu().numpy()
            assert got.shape == ref.shape
            for sl in (slice(0, 3), slice(3, 4), slice(4, None)):
                assert scale_err(got[:, sl], ref[:, sl]) <= tol, (impl, m, ins_num, scale_err(got[:, sl], ref[:, sl]))
        ref64 = O.mlp_forward(O.to_torch(w, torch.float64), x.double()).numpy()
        got = net(_cu(x), impl=_lib.IMPL_UMMA_F16).cpu().numpy()
        assert got.shape == ref64.shape and np.isfinite(got).all()
        assert rel_l2(got, ref64) <= 2e-3, (m, ins_num, rel_l2(got, ref64))


@settings(**COMMON)
@given(n=st.integers(5, 400), k=st.integers(2, 128), seed=st.integers(0, 2 ** 20), frac_present=st.floats(0.2, 1.0))
def test_hungarian_loss_fuzz(n, k, seed, frac_present):
    """Hungarian-matched instance loss (evaluator.py:19-74) at random batch sizes / channel counts / label subsets: loss parts
    and the gradient w.r.t. the instance map against the oracle (which is pinned bit for bit to the reference)."""
    from dmnerf_b200.evaluator import ins_criterion
    gen = torch.Generator().manual_seed(seed)
    n_present = max(1, min(k, int(round(frac_present * min(k, n)))))
    present = torch.randperm(k, generator=gen)[:n_present]
    lab = present[torch.randint(0, n_present, (n,), generator=gen)].float()
    logits = torch.randn(n, k, generator=gen) * 2
    logits[torch.arange(n), lab.long()] += 3.0
    pred = torch.sigmoid(logits)
    p_ref = pred.clone().requires_grad_(True)
    ref = O.ins_criterion(p_ref, lab, k)
    ref[0].sum().backward()
    p_gpu = _cu(pred).requires_grad_(True)
    got = ins_criterion(p_gpu, _cu(lab), k)
    got[0].sum().backward()
    for a, b in zip(got, ref):
        assert abs(float(a.detach().float().sum()) - float(b.detach().float().sum())) <= 2e-5 * max(1.0, abs(float(b.detach().float().sum())))
    g_ref = p_ref.grad.numpy()
    g_got = p_gpu.grad.cpu().numpy()
    scale = max(float(np.abs(g_ref).max()), 1e-12)
    assert float(np.abs(g_got - g_ref).max()) <= 2e-5 * scale, (n, k, n_present)


@settings(**COMMON)
@given(n=st.integers(1, 40), s=st.integers(3, 200), k=st.integers(2, 128), seed=st.integers(0, 2 ** 20))
def test_penalizer_fuzz(n, s, k, seed):
    """Emptiness penalizer (penalizer.py:5-62) at ragged sizes and every shared-memory tile size of the kernels (C <= 48, <= 96,
    <= 132): value and gradient against the oracle."""
    import types
    from dmnerf_b200.penalizer import ins_penalizer
    gen = torch.Generator().manual_seed(seed)
    # |logit| <~ 4: d/dx -log(1 - sigmoid(x)) = sigmoid'(x) / (1 - sigmoid(x)) amplifies the last bit of the sigmoid by
    # 1 / (1 - p); larger logits would test the conditioning of that quotient (the same in the reference), not the kernels
    raw = torch.randn(n, s, 4 + k, generator=gen).clamp(-4.0, 4.0)
    z = torch.rand(n, s, generator=gen).sort(-1).values * 11 + 4
    rd = torch.randn(n, 3, generator=gen) * 1.3
    depth = z[torch.arange(n), torch.randint(0, s, (n,), generator=gen)] + 0.01
    r_ref = raw.clone().requires_grad_(True)
    ref = O.ins_penalizer(r_ref, z, depth, rd, 0.05, 0.05)
    ref.sum().backward()
    r_gpu = _cu(raw).requires_grad_(True)
    got = ins_penalizer(r_gpu, _cu(z), _cu(depth), _cu(rd), types.SimpleNamespace(tolerance=0.05, deta_w=0.05))
    got.sum().backward()
    assert abs(float(got.detach().sum()) - float(ref.detach().sum())) <= 2e-5 * max(1e-6, abs(float(ref.detach().sum())))
    g_ref, g_got = r_ref.grad.numpy(), r_gpu.grad.cpu().numpy()
    scale = max(float(np.abs(g_ref).max()), 1e-12)
    assert float(np.abs(g_got - g_ref).max()) <= 5e-5 * scale and float(np.abs(g_got[..., :4]).max()) == 0.0, \
        (float(np.abs(g_got - g_ref).max()), scale)
