"""fp64 restatements of the training step's loss kernels, with first-order fp32 rounding budgets -- TEST INFRASTRUCTURE ONLY
(same standing as oracle/dmnerf_oracle.py; the product package never imports it).

Each function is fed a kernel's exact fp32 inputs.  Every discrete decision is taken by the fp32 rule of the library, so it is
the kernel's decision: a sample's object label (argmax of the fp32 sigmoid, first maximum), a penalizer mask (the kernel's fp32
formulas for |d|, front, back and position), the assignment (given).  Only the arithmetic runs in fp64 (or in `dtype`: run in
float32, a restatement takes the fp32 oracle's own steps).

A budget bounds |fp32 result - fp64 result| element by element.  It is a first-order rounding analysis evaluated in fp64 on the
same inputs, with u = 2^-24 the unit roundoff of fp32:
  composite  `1 - exp(-x)` costs 4u e + u alpha on alpha (expf is within 2 ulp) plus the propagated 6u relative error of x
             (the z difference, |d|, the products); every transmittance factor f = 1 - alpha + 1e-10 is taken at the top of its
             error interval, and the product of those, with (i + 2) u for the roundings of transmittance i, bounds it; a
             weighted sum of S terms costs (S + 1) u sum|terms| on top of its terms' errors; the fp32 sigmoid costs 6u relative.
  penalizer  every -log(q) term, q = 1 - p + 1e-8 or p + 1e-8, is charged its condition number: dq / q; the gaussian its
             argument's error; the kernel adds its per-sample fp32 terms in fp64 (no summation charge beyond K + 1 ulp per
             sample), the fp32 oracle sums in fp32 (charged 2 log2(M) + 8 ulp of sum|terms| over M terms).
  instance   the log terms as in the penalizer, fp64 sums, then the fp32 evaluation of cost_siou as the kernel writes it.
The budgets are validated against the fp32 oracles (the reference's own arithmetic) in tests/test_fp64_budget_host.py before a
kernel is held to them."""
import math

import numpy as np
import torch

from . import appearance_oracle as AO
from . import dmnerf_oracle as O
from . import objects_oracle as OO
from . import region_oracle as RO

U = 2.0 ** -24
SATURATED = 17.0          # sigmoid(x) rounds to exactly 1.0f for x above ~16.7 whatever the exp's last bit


# ------------------------------------------------------------------------------------------------------------ labels
def labels32(raw):
    """The library's label of every sample, from the fp32 logits raw[..., 4:]: argmax of the fp32 sigmoid, first maximum."""
    return OO.object_labels(raw.float())


def near_tie(raw):
    """Bool [...]: the label could flip with the last bit of an implementation's sigmoid.  A sample is flagged when a channel
    whose logit differs from the winner's has an fp32 sigmoid within 2 ulp of the winner's (identical logits are exact ties,
    which the first-maximum rule settles the same way everywhere; two logits that both saturate to 1.0f are too)."""
    lg = raw.float()[..., 4:]
    sig = torch.sigmoid(lg)
    lab = torch.argmax(sig, -1, keepdim=True)
    top, top_lg = torch.gather(sig, -1, lab), torch.gather(lg, -1, lab)
    ulp2 = 2.0 * (top - torch.nextafter(top, torch.zeros_like(top)))
    close = (top - sig).abs() <= ulp2
    both_saturated = (lg >= SATURATED) & (top_lg >= SATURATED)
    return (close & (lg != top_lg) & ~both_saturated).any(-1)


def _edited(raw, z, keep, exclude):
    """(fp32 raw, fp32 labels, fp32 raw with the selection and the exclusion applied: zeroed densities are exact)."""
    r32 = raw.float()
    return r32, OO.object_labels(r32), RO._selected(r32, keep, z, exclude)


# ------------------------------------------------------------------------------------------------------------ composite
def composite64(raw, z, rays_d, keep_all_ins, keep=None, exclude=None, appearance=None, dtype=torch.float64):
    """The stage composite (networks/render.py:6-28, with the selection keep (bool [ins_num + 1]), the region's exclusion
    ((z, labels) -> bool) and the appearance of the library's select path) in `dtype` on fp32 inputs.  Returns a dict:
    rgb, weights, depth, ins, acc; labels (fp32 rule); near (near_tie); carries (weight > 0)."""
    r32, lab, sel = _edited(raw, z, keep, exclude)
    r, zz, rd = r32.to(dtype), z.float().to(dtype), rays_d.float().to(dtype)
    sel = sel.to(dtype)
    S = zz.shape[-1]
    if S == 1:
        # render.py:10 takes the 1e10 tail from dists[..., :1], which is empty for one sample; the library gives that sample
        # the tail: a second sample 1e10 further on with density 0 (alpha 0) does the same here and is dropped after
        pad = torch.zeros_like(sel)
        sel, r = torch.cat([sel, pad], -2), torch.cat([r, pad], -2)
        lab = torch.cat([lab, lab], -1)
        zz = torch.cat([zz, zz + 1e10], -1)
    if appearance is None:
        rgb, w, depth, ins, acc = O.composite(sel, zz, rd, keep_all_ins=keep_all_ins)
    else:
        rgb, w, depth, ins, acc = O.composite(AO.scale_density(sel, lab, appearance), zz, rd, keep_all_ins=keep_all_ins)
        rgb = torch.sum(w[..., None] * AO.edited_colour(r, lab, appearance), -2)
    w = w[..., :S]
    return {"rgb": rgb, "weights": w, "depth": depth, "ins": ins, "acc": acc, "labels": lab[..., :S], "near": near_tie(raw),
            "carries": w > 0}


def composite_budget(raw, z, rays_d, keep_all_ins, keep=None, exclude=None, appearance=None):
    """Per-element bound on |fp32 composite - composite64| for rgb, weights, depth, ins, acc (fp64 tensors)."""
    r32, lab, sel = _edited(raw, z, keep, exclude)
    r, sel, zz = r32.double(), sel.double(), z.float().double()
    rd = rays_d.float().double()
    sg = torch.relu(sel[..., 3])
    rx = 6.0 * U                                                   # z difference, |d| (3 rounded terms and a sqrt), 2 products
    if appearance is not None:
        table = AO._table(appearance, r)
        sg = table[:, 12][lab.to(r.device)] * sg
        rx += U
    S = zz.shape[-1]
    dist = torch.cat([zz[..., 1:] - zz[..., :-1], torch.full_like(zz[..., :1], 1e10)], -1)
    x = sg * dist * torch.norm(rd, dim=-1, keepdim=True)
    e = torch.exp(-x)
    alpha = 1.0 - e
    d_alpha = e * x * rx + 4.0 * U * e + U * alpha
    f = e + 1e-10
    d_f = d_alpha + U * e + U * f
    # the exclusive product of f (i factors, i + 2 roundings) can only grow to the product of the factors at the top of their
    # error intervals, f + df + u f; evaluated as a product (in log space, so that a run of saturated samples -- f = 1e-10 --
    # underflows to 0 instead of overflowing a relative error), the bound stays finite and 0 where the transmittance is
    excl = lambda t: torch.cat([torch.zeros_like(t[..., :1]), torch.cumsum(t, -1)[..., :-1]], -1)
    trans = torch.exp(excl(torch.log(f)))
    trans_hi = torch.exp(excl(torch.log(f + d_f + U * f)) + 2.0 * U)
    w = alpha * trans
    d_w = d_alpha * trans + alpha * (trans_hi - trans) + U * w + 2.0 ** -126        # the floor: fp32 denormals
    sum_u = (S + 1) * U
    out = {"weights": d_w, "acc": d_w.sum(-1) + sum_u * w.sum(-1)}
    out["depth"] = (d_w * zz.abs()).sum(-1) + sum_u * (w * zz.abs()).sum(-1)
    c = torch.sigmoid(r[..., :3])
    d_c = 6.0 * U * c
    if appearance is not None:
        m = table[:, :12].reshape(-1, 3, 4)[lab.to(r.device)]
        mc = (m[..., :3].abs() * c[..., None, :]).sum(-1)          # [..., 3]: sum_b |M_ab| c_b
        d_c = (m[..., :3].abs() * d_c[..., None, :]).sum(-1) + 4.0 * U * (mc + m[..., 3].abs())
        c = AO.edited_colour(r, lab, appearance)
    out["rgb"] = (d_w[..., None] * c + w[..., None] * d_c).sum(-2) + sum_u * (w[..., None] * c).sum(-2)
    lg = r[..., 4:] if keep_all_ins else r[..., 4:-1]
    a = (w[..., None] * lg).sum(-2)
    d_a = (d_w[..., None] * lg.abs()).sum(-2) + sum_u * (w[..., None] * lg.abs()).sum(-2)
    s = torch.sigmoid(a)
    out["ins"] = s * (1.0 - s) * d_a + 6.0 * U * s
    return out


# ------------------------------------------------------------------------------------------------------------ penalizer
def pen_masks(z, depth, rays_d, tol):
    """(before, middle) bool [N, S] by the kernel's fp32 formulas: norm = sqrt((d0^2 + d1^2) + d2^2), front = (depth - tol) norm,
    back = (depth + tol) norm, pos = z norm, every operation rounded once (penalizer.py:13-29)."""
    d = rays_d.float()
    norm = torch.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])[:, None]
    dep = depth.float().reshape(-1, 1)
    t = torch.tensor(float(np.float32(tol)), dtype=torch.float32, device=dep.device)
    front, back = (dep - t) * norm, (dep + t) * norm
    pos = z.float() * norm
    before, after = pos < front, pos > back
    return before, ~(before | after)


def penalizer64(raw, z, depth, rays_d, tol, w, g_loss=1.0, dtype=torch.float64):
    """The emptiness penalizer (penalizer.py:5-55, O.emptiness_penalizer's steps) in `dtype` on fp32 inputs, with the kernel's
    fp32 masks.  Returns (loss [1], d loss / d raw * g_loss [N, S, C], (before, middle))."""
    before, middle = pen_masks(z, depth, rays_d, tol)
    r = raw.float().to(dtype).detach().requires_grad_(True)
    zz, dep = z.float().to(dtype), depth.float().reshape(-1, 1).to(dtype)
    sigma_h = torch.tensor([0.4], dtype=torch.float32).to(dtype)
    sigma_w = torch.tensor([w], dtype=torch.float32).to(dtype)
    two_pi_root = torch.sqrt(torch.tensor([2 * np.pi], dtype=torch.float32).to(dtype))
    if dtype != torch.float32:
        sigma_h, two_pi_root = torch.tensor([0.4], dtype=dtype), torch.sqrt(torch.tensor([2 * np.pi], dtype=dtype))
    dev = r.device
    sigma_h, sigma_w, two_pi_root = sigma_h.to(dev), sigma_w.to(dev), two_pi_root.to(dev)
    norm = torch.norm(rays_d.float().to(dtype)[..., None, :], dim=-1)                          # :13   [N, 1]
    surface, pos = dep * norm, zz * norm
    g = torch.exp(-((surface - pos) ** 2) / (2 * (sigma_w ** 2))) / (sigma_h * two_pi_root) + 1e-8
    air = 1 - g
    m_before, m_middle = before.to(dtype), middle.to(dtype)
    pred = torch.sigmoid(r[..., 4:])
    gt = torch.zeros_like(pred)
    gt[..., -1] = 1
    l_before = -gt * torch.log(pred + 1e-8) - (1 - gt) * torch.log(1 - pred + 1e-8)
    l_before = l_before * (air * m_before)[..., None]
    one_e8 = torch.tensor([1e-8], dtype=dtype, device=dev)
    l_before = torch.sum(l_before) / (pred.shape[-1] * torch.maximum(torch.sum(m_before), one_e8))
    last = pred[..., -1]
    l_mid = -torch.log(1 - last + 1e-8) * (g * m_middle)
    l_mid = torch.sum(l_mid) / torch.maximum(torch.sum(m_middle), one_e8)
    loss = l_before + l_mid
    (grad,) = torch.autograd.grad(loss.sum(), r)
    return loss.detach(), grad * float(g_loss), (before, middle)


def _log_terms(p):
    """(-log(1 - p + 1e-8), its bound, -log(p + 1e-8), its bound) for exact p with an fp32 error of 6u p: each term is
    charged its condition number (the error of q over q), plus 2 ulp of the log."""
    d_p = 6.0 * U * p
    q0, q1 = 1.0 - p + 1e-8, p + 1e-8
    d_q0 = d_p + U * (1.0 - p) + U * q0
    d_q1 = d_p + U * q1
    t0, t1 = -torch.log(q0), -torch.log(q1)
    dt0 = d_q0 / (q0 - d_q0).clamp(min=0.5e-8) + 2.0 * U * t0.abs()
    dt1 = d_q1 / (q1 - d_q1).clamp(min=0.5e-8) + 2.0 * U * t1.abs()
    return t0, dt0, t1, dt1


def _gaussian_budget(z, depth, rays_d, w):
    """(g, its bound) of the penalizer's gaussian (penalizer.py:7-8, 18-23) in fp64 on fp32 inputs."""
    d = rays_d.float().double()
    norm = torch.norm(d, dim=-1, keepdim=True)
    dep = depth.float().double().reshape(-1, 1)
    zz = z.float().double()
    surf, pos = dep * norm, zz * norm
    dd = surf - pos
    d_dd = U * (surf.abs() + pos.abs()) + 4.0 * U * dd.abs()
    w = float(np.float32(w))
    a = dd * dd / (2.0 * w * w)
    d_a = dd.abs() * d_dd / (w * w) + 4.0 * U * a
    den = 0.4 * math.sqrt(2.0 * math.pi)
    E = torch.exp(-a)
    g = E / den + 1e-8
    d_g = E * (d_a + 4.0 * U) / den + 4.0 * U * E / den + U * g
    return g, d_g


def penalizer_budget(raw, z, depth, rays_d, tol, w, g_loss=1.0, fp32_sums=False):
    """(bound on the loss, per-element bound on d raw) of penalizer64, for the kernel (fp32 terms per sample, fp64 sums) or,
    fp32_sums=True, for the fp32 oracle (every sum in fp32)."""
    before, middle = pen_masks(z, depth, rays_d, tol)
    r = raw.float().double()
    p = torch.sigmoid(r[..., 4:])
    K = p.shape[-1]
    t0, dt0, t1, dt1 = _log_terms(p)
    g, d_g = _gaussian_budget(z, depth, rays_d, w)
    air, d_air = 1.0 - g, d_g + U * (1.0 - g)
    last = torch.zeros(K, dtype=torch.bool, device=r.device)
    last[-1] = True
    t = torch.where(last, t1, t0)
    dt = torch.where(last, dt1, dt0)
    mb, mm = before.double(), middle.double()
    nb, nm = max(float(mb.sum()), 1e-8), max(float(mm.sum()), 1e-8)
    per_b = (dt * air[..., None] + t * d_air[..., None]).sum(-1) + (K + 1) * U * (t * air[..., None]).sum(-1)
    mid = g * t0[..., -1]
    per_m = d_g * t0[..., -1] + g * dt0[..., -1] + U * mid
    loss_b, loss_m = float((mb * air * t.sum(-1)).sum()) / (K * nb), float((mm * mid).sum()) / nm
    d_loss = float((mb * per_b).sum()) / (K * nb) + float((mm * per_m).sum()) / nm + 2.0 * U * (loss_b + loss_m)
    if fp32_sums:
        M = max(int(mb.sum()) * K, 1)
        d_loss += (2 * math.log2(M + 1) + 8) * U * loss_b + (2 * math.log2(max(int(mm.sum()), 1) + 1) + 8) * U * loss_m
    # gradient: h0 = p (1 - p) / (1 - p + eps) (the non-last classes and the middle term), h1 = p (1 - p) / (p + eps)
    # Both are increasing in p and in y = 1 - p (the kernel rounds each separately), so their error is bounded by evaluating them
    # at the ends of the intervals p +- dp, y +- dy: exact in each variable, where a tangent would fall short once p rounds to 1
    # (y = 0 in fp32 against y ~ 6e-8 in fp64 moves h0 = y / (y + eps) by far more than its slope at y predicts).
    eps = 1e-8
    y = 1.0 - p
    d_p = 6.0 * U * p
    d_y = d_p + U * y
    p_lo, p_hi = (p - d_p).clamp(min=0.0), p + d_p
    y_lo, y_hi = (y - d_y).clamp(min=0.0), y + d_y
    h0, h1 = p * y / (y + eps), p * y / (p + eps)
    spread = lambda h, lo, hi: torch.maximum(hi - h, h - lo)
    # + 3u: the product p (1 - p), the sum q = 1 - p + 1e-8 (or p + 1e-8) and the quotient dp / q
    d_h0 = spread(h0, p_lo * y_lo / (y_lo + eps), p_hi * y_hi / (y_hi + eps)) + 3.0 * U * h0
    d_h1 = spread(h1, p_lo * y_lo / (p_lo + eps), p_hi * y_hi / (p_hi + eps)) + 3.0 * U * h1
    cb, cm = abs(float(g_loss)) / (K * nb), abs(float(g_loss)) / nm
    h, dh = torch.where(last, h1, h0), torch.where(last, d_h1, d_h0)
    # + 4u: the scale (float)(1 / (K n)) and its product with g_loss, then (scale * air or g) and its product with h
    d_before = cb * (d_air[..., None] * h + air[..., None] * dh + 4.0 * U * air[..., None] * h)
    d_mid = cm * (d_g * h0[..., -1] + g * d_h0[..., -1] + 4.0 * U * g * h0[..., -1])
    d_grad = torch.zeros_like(r)
    d_grad[..., 4:] = d_before * mb[..., None]
    d_grad[..., -1] += d_mid * mm
    return d_loss, d_grad


# ------------------------------------------------------------------------------------------------------------ instance loss
def label_rows(labels, k):
    """(row of every ray: rank of its label among the distinct labels, ascending (torch.unique order, evaluator.py:21-25),
    number of distinct labels)."""
    valid = torch.unique(labels.long())
    return torch.searchsorted(valid, labels.long()), int(valid.numel())


def ins_loss64(pred, labels, k, row_of_col, g3=(1.0, 1.0, 1.0), dtype=torch.float64):
    """The Hungarian instance loss (evaluator.py:19-74) in `dtype` on fp32 pred [N, k], for the GIVEN assignment row_of_col [k]
    (matched row per prediction column, -1 unmatched).  The one-hot broadcast is collapsed to per-row sums.  Returns a dict:
    gt_row, row_count, cost_ce, cost_siou, tp, col_sum [k, k] / [k], losses (valid_ce, invalid_ce, valid_siou),
    d_pred = d (g3 . losses) / d pred."""
    n = pred.shape[0]
    dev = pred.device
    gt_row, V = label_rows(labels.to(dev), k)
    v = pred.float().to(dtype).detach().requires_grad_(True)
    gt = torch.zeros(n, k, dtype=dtype, device=dev)
    gt[torch.arange(n, device=dev), gt_row] = 1.0
    l1, l0 = torch.log(v + 1e-8), torch.log(1 - v + 1e-8)
    A = l0.sum(0)                                                     # [k]        sum_n log(1 - pred + 1e-8)
    B, C = gt.t() @ l1, gt.t() @ l0                                   # [k(g), k(p)]
    cost_ce = -(B + A[None, :] - C) / n                               # evaluator.py:57
    tp = gt.t() @ v
    col_sum, cnt = v.sum(0), gt.sum(0)
    fp, fn = col_sum[None, :] - tp, cnt[:, None] - tp
    cost_siou = 1.0 - tp / (tp + fp + fn + 1e-6)                      # evaluator.py:60-64
    roc = torch.as_tensor(row_of_col, device=dev).long()
    cols = torch.nonzero(roc >= 0).flatten()
    rows = roc[cols]
    valid_ce = cost_ce[rows, cols].mean()
    valid_siou = cost_siou[rows, cols].mean()
    un = torch.nonzero(roc < 0).flatten()
    invalid_ce = v[:, un].mean() if len(un) else torch.zeros((), dtype=dtype, device=dev)   # evaluator.py:30-33
    total = g3[0] * valid_ce + g3[1] * invalid_ce + g3[2] * valid_siou
    (d_pred,) = torch.autograd.grad(total, v)
    det = lambda t: t.detach()
    return {"gt_row": gt_row, "n_valid": V, "row_count": det(cnt), "cost_ce": det(cost_ce), "cost_siou": det(cost_siou),
            "tp": det(tp), "col_sum": det(col_sum), "losses": torch.stack([det(valid_ce), det(invalid_ce), det(valid_siou)]),
            "d_pred": d_pred}


def _rounding(x, d_in):
    """The rounding of an fp32 operation whose exact result is x (fp64) and whose operands carry d_in: none when x is an fp32
    value and the operands are exact, else u |x|."""
    exact = (x == x.float().double()) & (d_in == 0)
    return torch.where(exact, torch.zeros_like(x), U * x.abs())


def ins_loss_budget(pred, labels, k, row_of_col, g3=(1.0, 1.0, 1.0), fp32_sums=False):
    """Bounds on |fp32 - ins_loss64| for cost_ce, cost_siou, tp, col_sum, losses and d_pred, for the kernel (fp32 terms, fp64
    sums, the fp32 evaluation of cost_siou and of the gradient) or, fp32_sums=True, the fp32 oracle (sums over the rays in
    fp32)."""
    ref = ins_loss64(pred, labels, k, row_of_col, g3)
    n = pred.shape[0]
    dev = pred.device
    v = pred.float().double()
    gt = torch.zeros(n, k, dtype=torch.float64, device=dev)
    gt[torch.arange(n, device=dev), ref["gt_row"]] = 1.0
    q0, q1 = 1.0 - v + 1e-8, v + 1e-8
    d_q0 = U * (1.0 - v) + U * q0
    t0, t1 = torch.log(q0), torch.log(q1)
    dt0 = d_q0 / (q0 - d_q0).clamp(min=0.5e-8) + 2.0 * U * t0.abs()
    dt1 = U + 2.0 * U * t1.abs()
    sum_u = (2 * math.log2(n + 1) + 8) * U if fp32_sums else 0.0
    dA = dt0.sum(0) + sum_u * t0.abs().sum(0)
    dB = gt.t() @ (dt1 + sum_u * t1.abs())
    dC = gt.t() @ (dt0 + sum_u * t0.abs())
    cost_ce, tp, S, cnt = ref["cost_ce"], ref["tp"], ref["col_sum"], ref["row_count"]
    d_ce = (dA[None, :] + dB + dC) / n + 2.0 * U * cost_ce.abs()
    # siou, as the kernel evaluates it in fp32 from the fp64 sums: an operation whose exact result is an fp32 value and whose
    # operands carry no error rounds nothing (pred of 0, 0.5 and 1 make every sum such a value)
    d_tp = _rounding(tp, sum_u * tp) + sum_u * tp
    d_S = _rounding(S, sum_u * S) + sum_u * S
    fp, fn = S[None, :] - tp, cnt[:, None] - tp
    d_fp = d_S[None, :] + d_tp
    d_fp = d_fp + _rounding(fp, d_fp)
    d_fn = d_tp + _rounding(fn, d_tp)
    d_den = d_tp + d_fp
    d_den = d_den + _rounding(tp + fp, d_den)
    d_den = d_den + d_fn
    d_den = d_den + _rounding(tp + fp + fn, d_den)
    den = tp + fp + fn + 1e-6
    d_den = d_den + U * den
    ratio = tp / den
    d_siou = d_tp / den + tp * d_den / den ** 2 + U * ratio + U * ref["cost_siou"].abs()
    roc = torch.as_tensor(row_of_col, device=dev).long()
    cols = torch.nonzero(roc >= 0).flatten()
    rows = roc[cols]
    un = torch.nonzero(roc < 0).flatten()
    L = ref["losses"].abs()
    d_losses = torch.stack([d_ce[rows, cols].mean() + 2 * U * L[0],
                            (d_S[un].sum() / (n * len(un)) if len(un) else torch.zeros((), dtype=torch.float64, device=dev))
                            + 2 * U * L[1],
                            d_siou[rows, cols].mean() + 2 * U * L[2]])
    # d_pred: matched column p of row g: g_ce dce / (V n) + g_siou dsi / V, dce = -1 / (v + eps) on the row, 1 / (1 - v + eps)
    # off it; dsi = -1 / D on the row, TP / D^2 off it (D = S + cnt - TP + 1e-6, evaluated in fp32 from the fp32 sums)
    V = ref["n_valid"]
    g_row = torch.full((k,), -1, dtype=torch.long, device=dev)
    g_row[cols] = rows
    on = gt[:, g_row.clamp(min=0)] > 0                                 # [n, k]: ray i is on column p's matched row
    Dm = (S + cnt[g_row.clamp(min=0)] - tp[g_row.clamp(min=0), torch.arange(k, device=dev)] + 1e-6)[None, :]
    TPm = tp[g_row.clamp(min=0), torch.arange(k, device=dev)][None, :]
    d_Dm = U * (2.0 * S + 2.0 * cnt[g_row.clamp(min=0)] + TPm[0] + Dm[0])[None, :] + d_S[None, :] + d_tp[g_row.clamp(min=0), torch.arange(k, device=dev)][None, :]
    dce = torch.where(on, 1.0 / q1, 1.0 / q0)
    dsi = torch.where(on, 1.0 / Dm, TPm / Dm ** 2)
    rel_dsi = torch.where(on, d_Dm / Dm + U, (U * TPm + d_tp[g_row.clamp(min=0), torch.arange(k, device=dev)][None, :]) / TPm.clamp(min=1e-300)
                          + 2.0 * d_Dm / Dm + 2.0 * U)
    term_ce = abs(g3[0]) * dce / (V * n)
    term_si = abs(g3[2]) * dsi / V
    d_matched = term_ce * 8.0 * U + term_si * (rel_dsi + 3.0 * U) + U * (term_ce + term_si)
    d_unmatched = torch.full_like(v, abs(g3[1]) / (n * max(k - V, 1)) * 3.0 * U)
    d_pred = torch.where((g_row >= 0)[None, :], d_matched, d_unmatched)
    return {"cost_ce": d_ce, "cost_siou": d_siou, "tp": d_tp, "col_sum": d_S, "losses": d_losses, "d_pred": d_pred}, ref


# ------------------------------------------------------------------------------------------------------------ edge-case inputs
def _untie(raw):
    """Make every near tie (near_tie) an exact one: the channels within 2 ulp of the winner take the winner's logit."""
    for _ in range(4):
        nt = near_tie(raw)
        if not bool(nt.any()):
            return raw
        lg = raw[..., 4:]
        sig = torch.sigmoid(lg)
        lab = torch.argmax(sig, -1, keepdim=True)
        top, top_lg = torch.gather(sig, -1, lab), torch.gather(lg, -1, lab)
        close = (top - sig).abs() <= 2.0 * (top - torch.nextafter(top, torch.zeros_like(top)))
        raw[..., 4:] = torch.where(close & nt[..., None], top_lg.expand_as(lg), lg)
    assert not bool(near_tie(raw).any())
    return raw


def composite_inputs(n, S, k, seed, device="cpu"):
    """fp32 (raw [n, S, 4 + k], z [n, S], rays_d [n, 3]) on the CPU with every edge of the composite: densities negative, zero,
    1e4 (saturating), 1e-30 (alpha rounds to 0) and ordinary; logits up to +-80 on a fifth of the samples; exact ties of the
    winning logit with another channel on a third; zero-width bins; a ray with rays_d = 0 (ray 1 when n > 2).  No near ties
    (near_tie): a sample's label is the same under any correctly rounded sigmoid."""
    gen = torch.Generator(device).manual_seed(seed)
    raw = torch.randn(n, S, 4 + k, generator=gen, device=device) * 3
    kind = torch.randint(0, 6, (n, S), generator=gen, device=device)
    d = raw[..., 3]
    d = torch.where(kind == 0, -d.abs(), d.abs() * 2)
    d = torch.where(kind == 1, torch.zeros_like(d), d)
    d = torch.where(kind == 2, torch.full_like(d, 1e4), d)
    d = torch.where(kind == 3, torch.full_like(d, 1e-30), d)
    raw[..., 3] = d
    big = torch.rand(n, S, generator=gen, device=device) < 0.2
    raw[..., 4:] = torch.where(big[..., None], (raw[..., 4:] * 25).clamp(-80, 80), raw[..., 4:])
    if k > 1:
        tie = torch.rand(n, S, generator=gen, device=device) < 0.33
        lab = torch.argmax(torch.sigmoid(raw[..., 4:]), -1)
        other = torch.randint(0, k, (n, S), generator=gen, device=device)
        val = torch.gather(raw[..., 4:], -1, lab[..., None])[..., 0]
        lg = raw[..., 4:].clone()
        lg.scatter_(-1, other[..., None], torch.where(tie, val, torch.gather(lg, -1, other[..., None])[..., 0])[..., None])
        raw[..., 4:] = lg
    z = torch.rand(n, S, generator=gen, device=device).sort(-1).values * 9 + 1
    if S > 2:
        same = torch.rand(n, S - 1, generator=gen, device=device) < 0.1
        z[:, 1:] = torch.where(same, z[:, :-1], z[:, 1:])
        z = torch.cummax(z, -1).values
    rd = torch.randn(n, 3, generator=gen, device=device) * 1.5
    if n > 2:
        rd[1] = 0.0
    return _untie(raw).contiguous(), z.contiguous(), rd.contiguous()


def keep_split(k, seed):
    """A selection (bool [k]) keeping about half the labels, label 0 and not label 1: many of the exact ties of
    composite_inputs fall between a kept and a dropped label, so the first-maximum rule decides whether the sample is seen."""
    gen = torch.Generator().manual_seed(seed)
    keep = torch.rand(k, generator=gen) < 0.5
    keep[0] = True
    if k > 1:
        keep[1] = False
    return keep


def penalizer_inputs(n, S, k, seed, case="mixed", device="cpu"):
    """fp32 (raw [n, S, 4 + k], z [n, S], depth [n], rays_d [n, 3]) and (tol, w).  case: "mixed" (depths inside the samples,
    logits up to +-4 and +-24 on a tenth: p rounds to 0 or 1), "before" (depth behind every sample: all before), "behind" (depth
    in front of every sample: none before, none middle), "boundary" (samples exactly on z = depth -+ tol in fp32, and in the
    middle shell), "zero_d" (rays_d = 0: every sample in the middle)."""
    gen = torch.Generator(device).manual_seed(seed)
    tol, w = 0.05, 0.05
    raw = (torch.randn(n, S, 4 + k, generator=gen, device=device) * 2).clamp(-4, 4)
    sat = torch.rand(n, S, 4 + k, generator=gen, device=device) < 0.1
    raw = torch.where(sat, torch.sign(raw) * 24.0, raw)
    z = torch.rand(n, S, generator=gen, device=device).sort(-1).values * 11 + 4
    rd = torch.randn(n, 3, generator=gen, device=device) * 1.3
    depth = z[torch.arange(n, device=device), torch.randint(0, S, (n,), generator=gen, device=device)] + 0.01
    if case == "before":
        depth = z[:, -1] + 1.0
    elif case == "behind":
        depth = z[:, 0] - 1.0
    elif case == "boundary":
        t = torch.tensor(tol, dtype=torch.float32, device=device)
        pick = torch.randint(0, 3, (n, S), generator=gen, device=device)
        on = torch.stack([depth[:, None] - t, depth[:, None] + t, depth[:, None]], -1).expand(n, S, 3)
        z = torch.gather(on, -1, pick[..., None])[..., 0].contiguous()
    elif case == "zero_d":
        rd = torch.zeros(n, 3, device=device)
    return raw.contiguous(), z.contiguous(), depth.contiguous(), rd.contiguous(), tol, w


def ins_inputs(n, k, seed, case="mixed"):
    """fp32 pred [n, k] in [0, 1] with exact 0, 0.5 and 1 entries, and int32 labels [n].  case: "one" (a single label),
    "k" (exactly k labels: every column matched), "sparse" (ids up to 65535), "runs" (labels in runs longer than a warp and a
    label held by a single ray), "exact" (as "runs" with pred in {0, 0.5, 1} only: every sum of the costs is an fp32 value),
    "mixed" (a few labels)."""
    gen = torch.Generator().manual_seed(seed)
    logits = torch.randn(n, k, generator=gen) * 2
    pred = torch.sigmoid(logits)
    pick = torch.rand(n, k, generator=gen)
    pred = torch.where(pick < 0.05, torch.zeros_like(pred), pred)
    pred = torch.where((pick >= 0.05) & (pick < 0.08), torch.ones_like(pred), pred)
    pred = torch.where((pick >= 0.08) & (pick < 0.1), torch.full_like(pred, 0.5), pred)
    if case == "exact":
        pred = torch.randint(0, 3, (n, k), generator=gen).float() * 0.5
    n_lab = {"one": 1, "k": min(k, n)}.get(case, max(1, min(k, n, 1 + seed % 7)))
    ids = torch.randperm(65536 if case == "sparse" else k, generator=gen)[:n_lab]
    if case == "sparse":
        ids[0] = 65535
    if case in ("runs", "exact"):
        lab = ids[(torch.arange(n) // 40) % n_lab]
        lab[n // 2] = ids[-1] if n_lab > 1 else ids[0]
    else:
        lab = ids[torch.randint(0, n_lab, (n,), generator=gen)]
        lab[:n_lab] = ids                                              # every label present
    return pred.contiguous(), lab.to(torch.int32).contiguous()
