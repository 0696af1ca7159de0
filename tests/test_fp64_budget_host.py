"""CPU: the fp64 restatements of the stage composite, the emptiness penalizer and the Hungarian instance loss
(oracle/fp64_oracle.py) and their fp32 rounding budgets.  Run in float32 a restatement takes the fp32 oracle's own steps, so it
equals that oracle; and the fp32 oracles -- the reference's own arithmetic -- sit inside their budgets against the fp64
restatements on CPU-sized versions of every edge case tests/test_gpu_training_losses_fp64.py puts to the kernels.  A budget a
kernel is held to is thereby shown to be achievable."""
import numpy as np
import pytest
import torch
from scipy.optimize import linear_sum_assignment

from oracle import dmnerf_oracle as O
from oracle import fp64_oracle as F
from oracle import objects_oracle as OO

MAPS = ("rgb", "weights", "depth", "ins", "acc")


def _worst(got, ref, budget):
    """max |got - ref| / budget over the elements (0 where both agree exactly); the budget must be finite everywhere."""
    assert bool(torch.isfinite(budget).all()), "budget not finite"
    err = (got.double() - ref.double()).abs()
    return float(torch.where(err > 0, err / budget, torch.zeros_like(err)).max()) if err.numel() else 0.0


def _exclude(z, labels):
    """A stand-in for a region's exclusion: the odd labels beyond depth 5."""
    return (torch.as_tensor(z) > 5.0) & (torch.as_tensor(labels) % 2 == 1)


# ------------------------------------------------------------------------------------------------------------ composite
@pytest.mark.parametrize("keep_all", [False, True])
@pytest.mark.parametrize("edit", ["none", "keep", "region", "appearance"])
@pytest.mark.parametrize("S,k", [(1, 2), (2, 1), (33, 29), (64, 2), (130, 5), (1024, 3)])
def test_composite_oracle_inside_its_budget(S, k, edit, keep_all):
    from dmnerf_b200 import objects as OB
    raw, z, rd = F.composite_inputs(5, S, k, seed=S * 31 + k)
    assert not bool(F.near_tie(raw).any())
    keep = F.keep_split(k, S) if edit in ("keep", "appearance") else None
    exclude = _exclude if edit == "region" else None
    app = None
    if edit == "appearance" and k >= 2:
        app = OB.Appearance(k - 1, colour={0: np.array([[0.0, 0.0, 1.2, 0.05], [0.0, 1.0, 0.0, -0.1], [0.8, 0.0, 0.0, 0.0]])},
                            density={0: 2.5, 1: 0.0})
    ref = F.composite64(raw, z, rd, keep_all, keep, exclude, app)
    twin = F.composite64(raw, z, rd, keep_all, keep, exclude, app, dtype=torch.float32)
    # float32 restatement = the fp32 oracles (labels, selection, appearance and composite) bit for bit
    sel = raw if keep is None else OO.select_objects(raw, keep)
    if exclude is not None:
        sel = F.RO.exclude_samples(sel, exclude(z, OO.object_labels(raw)))
    oracle = F.AO.composite(raw, sel, z, rd, app, keep_all)
    assert torch.equal(ref["labels"], OO.object_labels(raw))
    for name, o in zip(MAPS, oracle):
        assert S == 1 or torch.equal(twin[name], o), name          # S = 1: the oracle has no tail distance (render.py:10)
    budget = F.composite_budget(raw, z, rd, keep_all, keep, exclude, app)
    worst = {m: _worst(twin[m], ref[m], budget[m]) for m in MAPS}
    print("\n  composite S %d k %d %s keep_all %d: fp32 oracle / budget %s" % (S, k, edit, keep_all,
          " ".join("%s %.3f" % kv for kv in worst.items())))
    assert all(v <= 1.0 for v in worst.values()), worst


def test_composite_first_maximum_wins_exact_ties():
    raw = torch.zeros(1, 3, 4 + 4)
    raw[..., 3] = 1.0
    raw[0, :, 4:] = torch.tensor([[1.0, 3.0, 3.0, 0.0], [30.0, 40.0, 50.0, 50.0], [-2.0, -2.0, -2.0, -2.0]])
    assert F.labels32(raw).tolist() == [[1, 0, 0]]                 # 30, 40, 50 all round to 1.0f: the first channel wins
    assert not bool(F.near_tie(raw).any())


# ------------------------------------------------------------------------------------------------------------ penalizer
@pytest.mark.parametrize("case", ["mixed", "before", "behind", "boundary", "zero_d"])
@pytest.mark.parametrize("n,S,k", [(1, 1, 1), (7, 33, 44), (5, 40, 93), (3, 20, 128)])
def test_penalizer_oracle_inside_its_budget(n, S, k, case):
    raw, z, depth, rd, tol, w = F.penalizer_inputs(n, S, k, seed=n + S + k, case=case)
    loss64, grad64, (before, middle) = F.penalizer64(raw, z, depth, rd, tol, w)
    loss32, grad32, masks32 = F.penalizer64(raw, z, depth, rd, tol, w, dtype=torch.float32)
    r = raw.clone().requires_grad_(True)
    oracle = O.emptiness_penalizer(r, z, depth[:, None], rd, tol, w)
    oracle.sum().backward()
    # the oracle takes its masks through torch.norm, which differs from the kernel's sqrt((d0^2 + d1^2) + d2^2) in the last bit
    # for some rays; none of these samples lies close enough to a mask boundary for that to move it, so the masks agree and
    # the float32 restatement (its gaussian through torch.norm too) is the oracle bit for bit
    d = rd.float()
    norm = torch.norm(d[..., None, :], dim=-1)
    pos, dep = z * norm, depth[:, None]
    assert torch.equal(before, pos < (dep - tol) * norm) and torch.equal(middle, ~((pos < (dep - tol) * norm) | (pos > (dep + tol) * norm)))
    assert torch.equal(loss32, oracle.detach()) and torch.equal(grad32, r.grad)
    if case == "before":
        assert bool(before.all())
    if case == "behind":
        assert not bool(before.any()) and not bool(middle.any())
    if case == "zero_d":
        assert bool(middle.all())
    if case == "boundary":
        assert bool(middle.any())
    d_loss, d_grad = F.penalizer_budget(raw, z, depth, rd, tol, w, fp32_sums=True)
    ol = float(oracle.detach())
    e_loss = abs(ol - float(loss64)) / d_loss if ol != float(loss64) else 0.0
    e_grad = _worst(r.grad, grad64, d_grad)
    print("\n  penalizer %dx%d k %d %s: fp32 oracle / budget loss %.3f grad %.3f" % (n, S, k, case, e_loss, e_grad))
    assert e_loss <= 1.0 and e_grad <= 1.0, (e_loss, e_grad)


# ------------------------------------------------------------------------------------------------------------ instance loss
@pytest.mark.parametrize("case", ["one", "k", "sparse", "runs", "exact", "mixed"])
@pytest.mark.parametrize("n,k", [(1, 1), (33, 2), (70, 13), (257, 33), (300, 127)])
def test_ins_loss_oracle_inside_its_budget(n, k, case):
    pred, labels = F.ins_inputs(n, k, seed=n * 7 + k, case=case)
    if len(torch.unique(labels)) > k:
        pytest.skip("more labels than channels")
    p = pred.clone().requires_grad_(True)
    total, vce, ice, vsi = O.ins_criterion(p, labels.float(), k)
    # the oracle's own assignment as row_of_col
    valid = torch.unique(labels.long())
    lab_cols = torch.searchsorted(valid, labels.long())
    gt = torch.zeros(n, k)
    gt[torch.arange(n), lab_cols] = 1.0
    cost_ce, cost_siou, order_row, order_col = O.hungarian(pred, gt, len(valid), k)
    roc = np.full(k, -1)
    roc[order_col[:len(valid)]] = order_row
    budget, ref = F.ins_loss_budget(pred, labels, k, roc, fp32_sums=True)
    assert torch.equal(ref["gt_row"], lab_cols) and ref["n_valid"] == len(valid)
    if ref["n_valid"] == k:
        assert float(ice.reshape(-1)[0]) == 0.0 and float(ref["losses"][1]) == 0.0   # every column matched: no invalid_ce
    total.sum().backward()
    worst = {"cost_ce": _worst(cost_ce, ref["cost_ce"], budget["cost_ce"]),
             "cost_siou": _worst(cost_siou, ref["cost_siou"], budget["cost_siou"]),
             "losses": _worst(torch.stack([vce.reshape(()), ice.reshape(()).float(), vsi.reshape(())]).detach(), ref["losses"],
                              budget["losses"]),
             "d_pred": _worst(p.grad, ref["d_pred"], budget["d_pred"])}
    # scipy on the fp32 costs is optimal on the fp64 costs to within k ulp of the largest cost
    sc32 = (cost_ce + cost_siou)[:len(valid)].numpy()
    r32, c32 = linear_sum_assignment(sc32)
    sc64 = (ref["cost_ce"] + ref["cost_siou"])[:len(valid)].numpy()
    r64, c64 = linear_sum_assignment(sc64)
    assert sc64[r32, c32].sum() - sc64[r64, c64].sum() <= k * 2.0 ** -23 * max(np.abs(sc64).max(), 1.0)
    print("\n  ins loss n %d k %d %s: fp32 oracle / budget %s" % (n, k, case, " ".join("%s %.3f" % kv for kv in worst.items())))
    assert all(v <= 1.0 for v in worst.values()), worst
