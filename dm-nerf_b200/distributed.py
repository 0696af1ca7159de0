"""Data-parallel training: one step over W processes that equals the one-process step on the same batch.

Every rank makes the original's draws at full size (pixels, then torch.rand([N, 64]), then torch.rand([N, 128])) and keeps its
contiguous row range (parallel.shard_range).  Rays are independent in the renderer, so the forward of a shard is the rows of
the one-process forward.  Three losses are ratios of sums over the whole batch, so they are split into a per-shard partial and
a merge that every rank evaluates on the same gathered partials, in rank order:

    ins_criterion_sharded   the Hungarian-matched instance loss (evaluator.py:19-74): label bitmaps, then fp64 cost sums
    ins_penalizer_sharded   the emptiness penalizer (penalizer.py:5-62): mask populations and masked sums
    img2mse_sharded         the colour loss (evaluator.py:11): the sum of squares

Each returns the global value, identical on every rank; its backward is the gradient of that value w.r.t. the rank's own
inputs and needs no collective.  train_iteration then all-reduces the 60 parameter gradients in one flat buffer, so every
replica takes the same Adam step.  DESIGN.md, "Data-parallel training", gives the merge order and the determinism argument.
"""
import torch

from .backward import render_rays_grad
from .engine import ordered_params
from .evaluator import _MatchedLossDevice, _check_status
from .parallel import all_gather, all_reduce_sum_, shard_range, world_of
from .penalizer import _Penalizer
from .render import reference_draws


def instance_rows(lo, hi, n_global, n_ins=None):
    """The instance loss covers the last n_ins rays of the batch (all of them when n_ins is None; get_select_crop puts the
    labelled pixels last).  For a rank holding global rows [lo, hi) -> (a, b, off): its instance rows are the global rows
    [a, b), i.e. rows [a - lo, b - lo) of its shard and rows [a - off, b - off) of the n_ins labels; empty when a == b."""
    off = n_global - (n_global if n_ins is None else n_ins)
    a = min(max(lo, off), hi)
    return a, hi, off


# ------------------------------------------------------------------------------------------------------------- instance loss
def ins_assignment_sharded(pred_ins, gt_labels, ins_num, n_global, group=None):
    """ins_criterion_sharded's terms plus the matching: (valid_ce, invalid_ce, valid_siou, n_valid [1], row_of_col [ins_num]),
    all on the device and identical on every rank."""
    if not pred_ins.is_cuda:
        raise RuntimeError("ins_criterion_sharded: expected CUDA tensors (no CPU fallback)")
    if pred_ins.dim() != 2 or pred_ins.shape[1] != ins_num or gt_labels.shape[0] != pred_ins.shape[0]:
        raise RuntimeError("ins_criterion_sharded: pred_ins %s / gt_labels %s / ins_num %d are inconsistent"
                           % (tuple(pred_ins.shape), tuple(gt_labels.shape), ins_num))
    _check_status(pred_ins.device, "ins_criterion_sharded")
    labels = gt_labels.to(pred_ins.device).reshape(-1).to(torch.int32).contiguous()
    return _MatchedLossDevice.apply(pred_ins, labels, int(n_global), group)


def ins_criterion_sharded(pred_ins, gt_labels, ins_num, n_global, group=None):
    """evaluator.ins_criterion over a batch of n_global rays of which this rank holds the rows pred_ins [n, ins_num] /
    gt_labels [n] (n may be 0: the rank still joins the collectives).  Returns (ins_loss_sum, valid_ce, invalid_ce, valid_siou)
    of the whole batch on every rank.  Rejected labels on any rank: NaN losses and zero gradients on every rank, and the next
    call raises on every rank."""
    valid_ce, invalid_ce, valid_siou, _, _ = ins_assignment_sharded(pred_ins, gt_labels, ins_num, n_global, group)
    return valid_ce + invalid_ce + valid_siou, valid_ce, invalid_ce, valid_siou


# ------------------------------------------------------------------------------------------------------------------ penalizer
def ins_penalizer_sharded(raw, z_vals, depth, rays_d, args, group=None):
    """penalizer.ins_penalizer over the whole batch (its mask populations count the samples of every rank) from this rank's
    rows: the loss [1] of the whole batch on every rank.  The penalizer needs no global ray count: its normalisers are the
    merged populations."""
    return _Penalizer.apply(raw, z_vals, depth[..., None].detach(), rays_d, args.tolerance, args.deta_w, group)


# ----------------------------------------------------------------------------------------------------------------- colour loss
class _MseSharded(torch.autograd.Function):
    @staticmethod
    def forward(fctx, x, y, n_global, group):
        d = x.detach().float() - y.detach().float().to(x.device)
        parts = all_gather((d * d).sum().reshape(1), group)                   # fp32 sum of squares per rank
        denom = float(n_global) * (d[0].numel() if d.dim() > 1 else 1)
        fctx.save_for_backward(d)
        fctx.denom = denom
        return (parts.double().sum() / denom).float()

    @staticmethod
    def backward(fctx, g):
        d, = fctx.saved_tensors
        return g * (2.0 / fctx.denom) * d, None, None, None


def img2mse_sharded(x, y, n_global, group=None):
    """evaluator.img2mse (the mean of (x - y)^2) over the n_global rows of the batch, from this rank's rows x, y."""
    return _MseSharded.apply(x, y, int(n_global), group)


# ------------------------------------------------------------------------------------------------------------ training step
def all_reduce_grads(params, group=None):
    """Sum the parameters' gradients over the ranks: one all-reduce of one flat buffer."""
    world, _ = world_of(group)
    if world == 1:
        return
    grads = [p.grad for p in params]
    flat = torch.cat([g.reshape(-1) for g in grads])
    all_reduce_sum_(flat, group)
    torch._foreach_copy_(grads, [v.view_as(g) for v, g in zip(flat.split([g.numel() for g in grads]), grads)])


def train_iteration(i, batch, model_coarse, model_fine, optimizer, args, z_vals_coarse, group=None):
    """One iteration of train_dmsr.py:23-75 (and of the crop loop of train_scannet.py) across the ranks of `group`.

    batch = (target_c [N,3], target_i, batch_rays [2,N,3], N_ins): the WHOLE batch, made identically on every rank (the same
    get_select_full / get_select_crop draws: seed numpy alike on every rank); N_ins = None for full selection, where target_i
    has N labels, or the crop's instance count, where target_i holds the labels of the last N_ins rays.  The uniforms of the
    perturbed render are drawn at full size too (seed torch alike on every rank) and every rank keeps its own rows.
    args: perturb, N_importance, ins_num, penalize, tolerance, deta_w, lrate, lrate_decay.  z_vals_coarse: z_val_sample(N, ...).

    Renders the rank's rows, evaluates the sharded losses, back-propagates, all-reduces the gradients, steps the optimizer and
    applies the original's learning-rate decay.  Returns a dict of the global loss values (device tensors, identical on every
    rank: "total", "rgb", "ins", "emptiness"), the matchings "row_of_col_coarse" / "row_of_col_fine", the rank's rows [lo, hi)
    and its forward maps "out"."""
    target_c, target_i, batch_rays, n_ins = batch
    world, rank = world_of(group)
    n = batch_rays.shape[1]
    lo, hi, _ = shard_range(n, world, rank)
    if hi <= lo:
        raise ValueError("train_iteration: %d rays cannot be split over %d ranks" % (n, world))
    dev = batch_rays.device
    perturb = float(args.perturb) if args.perturb else 0.0
    t_rand, u = reference_draws(perturb, n, z_vals_coarse.shape[-1], args.N_importance, dev)
    rows = slice(lo, hi)
    out = render_rays_grad(batch_rays[0, rows], batch_rays[1, rows], model_coarse, model_fine, z_vals_coarse[rows], perturb,
                           args.N_importance, None if t_rand is None else t_rand[rows], None if u is None else u[rows])
    a, b, off = instance_rows(lo, hi, n, n_ins)
    n_ins_global = n - off
    labels = target_i[a - off:b - off]
    rgb_c = img2mse_sharded(out["rgb_coarse"], target_c[rows], n, group)
    ins_c = ins_assignment_sharded(out["ins_coarse"][a - lo:b - lo], labels, args.ins_num, n_ins_global, group)
    rgb_f = img2mse_sharded(out["rgb_fine"], target_c[rows], n, group)
    ins_f = ins_assignment_sharded(out["ins_fine"][a - lo:b - lo], labels, args.ins_num, n_ins_global, group)
    ins_loss = (ins_f[0] + ins_f[1] + ins_f[2]) + (ins_c[0] + ins_c[1] + ins_c[2])
    rgb_loss = rgb_f + rgb_c
    total = ins_loss + rgb_loss
    res = {"rgb": rgb_loss, "ins": ins_loss, "row_of_col_coarse": ins_c[4], "row_of_col_fine": ins_f[4], "lo": lo, "hi": hi,
           "out": out}
    if args.penalize:
        rays_d = batch_rays[1, rows]
        emptiness = ins_penalizer_sharded(out["raw_fine"], out["z_vals_fine"], out["depth_fine"], rays_d, args, group) \
            + ins_penalizer_sharded(out["raw_coarse"], out["z_vals_coarse"], out["depth_coarse"], rays_d, args, group)
        total = total + emptiness
        res["emptiness"] = emptiness
    optimizer.zero_grad()
    total.sum().backward()
    params = ordered_params(model_coarse)[0] + ordered_params(model_fine)[0]
    all_reduce_grads(params, group)
    optimizer.step()
    new_lrate = args.lrate * (0.1 ** (i / (args.lrate_decay * 1000)))          # train_dmsr.py:66-71
    for param_group in optimizer.param_groups:
        param_group["lr"] = new_lrate
    res["total"] = total
    return res


def replicas_identical(params, group=None):
    """True when every rank holds bit-identical `params`: one all-gather of a two-word fingerprint of their bits (a cheap check
    a trainer can run every i_print steps)."""
    bits = torch.cat([p.detach().reshape(-1) for p in params]).view(torch.int32).to(torch.int64)
    weight = torch.arange(bits.numel(), device=bits.device, dtype=torch.int64) * 2 + 1
    fp = torch.stack([bits.sum(), (bits * weight).sum()])
    every = all_gather(fp, group)
    return bool((every == every[0]).all())
