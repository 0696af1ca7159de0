"""networks/evaluator.py:19-74 on the native kernels: the Hungarian-matched instance loss of the training step.

    ins_criterion(pred_ins, gt_labels, ins_num) -> (ins_loss_sum, valid_ce, invalid_ce, valid_siou)     evaluator.py:19-37
    hungarian(pred_ins, gt_ins, valid_ins_num, ins_num) -> (cost_ce, cost_siou, order_row, order_col)   evaluator.py:41-74
    img2mse, mse2psnr, to8b                                                                             evaluator.py:11,14,15

The two [ins x ins] cost matrices come out of ONE pass over the rays (csrc/evaluator.cu: gt is one-hot, so the reference's
[ins x ins x N] broadcast collapses to per-row sums, added in an order fixed by the batch size: the costs, the matching and the
gradient are reproducible bit for bit).  ins_criterion then runs the assignment ON THE DEVICE (scipy's
shortest-augmenting-path algorithm restated for one warp, same fp64 duals and tie rule: the training iteration has no
device->host hop left; DMNERF_INS_ASSIGN=host selects scipy on the host, the reference's own arrangement, with one hop per
call).  hungarian() returns the reference's numpy orders and therefore always uses scipy.  The matched loss and its gradient
w.r.t. the rendered instance map are evaluated on the device (dmnerf_hungarian_assign / dmnerf_ins_loss_backward).

The device path is one autograd Function for one process and for a batch split over the ranks of a process group
(distributed.ins_criterion_sharded): one process is the one-shard case, whose costs equal the merge of one shard's partials
bit for bit.
"""
import os
import numpy as np
import torch

from . import _lib
from .engine import get_context
from .parallel import all_gather, world_of

img2mse = lambda x, y: torch.mean((x - y) ** 2)                                        # evaluator.py:11
to8b = lambda x: (255 * np.clip(x, 0, 1)).astype(np.uint8)                              # evaluator.py:14
mse2psnr = lambda x: -10. * torch.log(x) / torch.log(torch.tensor([10.], device=x.device))   # evaluator.py:15


def _cost_buffers(k, dev):
    e = lambda *s: torch.empty(s, device=dev, dtype=torch.float32)
    return {"cost_ce": e(k, k), "cost_siou": e(k, k), "tp": e(k, k), "col_sum": e(k), "row_count": e(k)}


def _cost_ptrs(c):
    return [_lib.ptr(c[key]) for key in ("cost_ce", "cost_siou", "tp", "col_sum", "row_count")]


def _costs(pred, gt_row):
    """pred [N,K] float32 contiguous, gt_row [N] int32 -> dict of device tensors (cost matrices + backward sums)."""
    n, k = pred.shape
    out = _cost_buffers(k, pred.device)
    get_context(pred.device).call("dmnerf_hungarian_costs", _lib.ptr(pred), _lib.ptr(gt_row, torch.int32), n, k, *_cost_ptrs(out))
    return out


def _loss_backward(saved, n_global, grads):
    """d (g_ce valid_ce + g_inv invalid_ce + g_siou valid_siou) / d pred for the rows pred [n,K] of a batch of n_global rays;
    saved = (pred, gt_row, row_of_col, n_valid [1] on the device, tp, col_sum, row_count), grads = (g_ce, g_inv, g_siou)."""
    pred, gt_row, row_of_col, n_valid, tp, col_sum, row_count = saved
    n, k = pred.shape
    zero = pred.new_zeros(())
    g3 = torch.stack([(g if g is not None else zero).reshape(()).float() for g in grads]).contiguous()
    d_pred = torch.empty_like(pred)
    i32 = torch.int32
    get_context(pred.device).call("dmnerf_ins_loss_backward", _lib.ptr(pred), _lib.ptr(gt_row, i32), n, n_global, k,
                                  _lib.ptr(row_of_col, i32), _lib.ptr(n_valid, i32), _lib.ptr(tp), _lib.ptr(col_sum),
                                  _lib.ptr(row_count), _lib.ptr(g3), _lib.ptr(d_pred))
    return d_pred


def _reorder(cost_matrix, valid_ins_num, ins_num):
    """evaluator.py:42-50 (host): assignment on the valid rows, unmatched prediction channels appended."""
    from scipy.optimize import linear_sum_assignment
    scores = cost_matrix[:valid_ins_num].detach().cpu().numpy()
    row_ind, col_ind = linear_sum_assignment(scores)
    if ins_num - valid_ins_num > 0:
        unmapped = np.array(list(set(range(ins_num)) - set(col_ind)))
        col_ind = np.concatenate([col_ind, unmapped])
    return row_ind, col_ind


def _rows_of_dense_gt(gt_ins):
    """Dense one-hot-or-zero gt_ins [N,K] -> row index per ray (-1 where the ray has no label)."""
    has = gt_ins.sum(-1) > 0
    return torch.where(has, gt_ins.argmax(-1), torch.full_like(has, -1, dtype=torch.int64)).to(torch.int32)


def hungarian(pred_ins, gt_ins, valid_ins_num, ins_num):
    """evaluator.py:41-74 for CUDA tensors (no gradient: use ins_criterion for the differentiable loss)."""
    if not pred_ins.is_cuda:
        raise RuntimeError("hungarian: expected CUDA tensors (no CPU fallback)")
    pred = pred_ins.detach().contiguous().float()
    gt_row = _rows_of_dense_gt(gt_ins.to(pred.device)).contiguous()
    c = _costs(pred, gt_row)
    order_row, order_col = _reorder(c["cost_ce"] + c["cost_siou"], valid_ins_num, ins_num)
    return c["cost_ce"], c["cost_siou"], order_row, order_col


class _MatchedLoss(torch.autograd.Function):
    """forward(pred_ins [N,K], gt_row [N] int32, valid_rows): gt_row[i] = cost-matrix row of ray i.  valid_rows = None: the rows
    are the label VALUES themselves (labels in [0, K)); which of them occur is read off the row populations that come back with
    the cost matrices -- ONE device->host hop per call.  valid_rows = n: rows 0..n-1 are the compacted labels (general path)."""

    @staticmethod
    def forward(fctx, pred_ins, gt_row, valid_rows):
        pred = pred_ins.detach().contiguous().float()
        n, k = pred.shape
        c = _costs(pred, gt_row)
        dev = pred.device
        if valid_rows is None:
            host = torch.cat([(c["cost_ce"] + c["cost_siou"]).reshape(-1), c["row_count"]]).cpu().numpy()   # the one sync
            scores_all, counts = host[:k * k].reshape(k, k), host[k * k:]
            if int(round(float(counts.sum()))) != n:
                raise _LabelsOutOfRange()
            rows_present = np.nonzero(counts > 0)[0]                                        # ascending = torch.unique order
            scores = scores_all[rows_present]
        else:
            rows_present = np.arange(int(valid_rows))
            scores = (c["cost_ce"] + c["cost_siou"])[:int(valid_rows)].cpu().numpy()
        n_valid = len(rows_present)
        from scipy.optimize import linear_sum_assignment
        row_ind, col_ind = linear_sum_assignment(scores)                                    # evaluator.py:45-47
        unmatched = np.array(sorted(set(range(k)) - set(col_ind.tolist())), dtype=np.int64)
        rows = torch.as_tensor(rows_present[row_ind], device=dev, dtype=torch.int64)
        cols = torch.as_tensor(col_ind, device=dev, dtype=torch.int64)
        valid_ce = c["cost_ce"][rows, cols].mean()                                          # evaluator.py:28
        valid_siou = c["cost_siou"][rows, cols].mean()                                      # evaluator.py:34
        row_of_col = torch.full((k,), -1, device=dev, dtype=torch.int32)
        row_of_col[cols] = rows.to(torch.int32)
        if len(unmatched):                                                                  # evaluator.py:30-33
            un = torch.as_tensor(unmatched, device=dev, dtype=torch.int64)
            invalid_ce = c["col_sum"][un].sum() / float(n * len(un))
        else:
            invalid_ce = torch.zeros((), device=dev)
        n_valid_dev = torch.tensor([int(n_valid)], device=dev, dtype=torch.int32)
        fctx.save_for_backward(pred, gt_row, row_of_col, n_valid_dev, c["tp"], c["col_sum"], c["row_count"])
        fctx.in_shape = pred_ins.shape
        n_valid_t = torch.tensor(int(n_valid))                                               # host-side by-product, not differentiable
        fctx.mark_non_differentiable(n_valid_t)
        return valid_ce, invalid_ce, valid_siou, n_valid_t

    @staticmethod
    def backward(fctx, g_ce, g_inv, g_siou, _g_n=None):
        saved = fctx.saved_tensors
        return _loss_backward(saved, saved[0].shape[0], (g_ce, g_inv, g_siou)).reshape(fctx.in_shape), None, None


class _LabelsOutOfRange(Exception):
    pass


class _MatchedLossDevice(torch.autograd.Function):
    """forward(pred_ins [n,K], labels [n] int32, n_global, group): ranks of the labels, cost matrices, assignment and the three
    loss terms of a batch of n_global rays, nothing read back.  One process (world 1, n = n_global): three launches.  Over the
    W ranks of `group`, each holding n rows of the batch: the label bitmaps and the fp64 cost partials are gathered and merged
    in rank order, so every rank gets the same costs, matching and losses.  Labels outside [0, 65536) or more distinct labels
    than K: NaN losses, zero gradient, and the next call raises (error word in mapped host memory)."""

    @staticmethod
    def forward(fctx, pred_ins, labels, n_global, group):
        pred = pred_ins.detach().contiguous().float()
        n, k = pred.shape
        dev = pred.device
        ctx = get_context(dev)
        world, _ = world_of(group)
        i32 = torch.int32
        gt_row = torch.empty(n, device=dev, dtype=i32)
        n_valid = torch.empty(1, device=dev, dtype=i32)
        if world == 1:
            if n != n_global:
                raise ValueError("instance loss: %d rows of a one-process batch of %d rays" % (n, n_global))
            ctx.call("dmnerf_ins_label_rows", _lib.ptr(labels, i32), n, k, _lib.ptr(gt_row, i32), _lib.ptr(n_valid, i32))
            c = _costs(pred, gt_row)
        else:
            bitmap = torch.empty(_lib.LABEL_WORDS, device=dev, dtype=i32)         # uint32 words in int32 storage
            ctx.call("dmnerf_ins_label_bitmap", _lib.ptr(labels, i32), n, _lib.ptr(bitmap, i32))
            bitmaps = all_gather(bitmap, group)
            ctx.call("dmnerf_ins_label_rows_merged", _lib.ptr(bitmaps, i32), world, _lib.ptr(labels, i32), n, k, _lib.ptr(gt_row, i32),
                     _lib.ptr(n_valid, i32))
            part = torch.empty(3 * k * (k + 1), device=dev, dtype=torch.float64)
            ctx.call("dmnerf_hungarian_partials", _lib.ptr(pred), _lib.ptr(gt_row, i32), n, k, _lib.ptr(part, torch.float64))
            parts = all_gather(part, group)
            c = _cost_buffers(k, dev)
            ctx.call("dmnerf_hungarian_costs_merged", _lib.ptr(parts, torch.float64), world, n_global, k, *_cost_ptrs(c))
        row_of_col = torch.empty(k, device=dev, dtype=i32)
        losses = torch.empty(3, device=dev, dtype=torch.float32)
        ctx.call("dmnerf_hungarian_assign", _lib.ptr(c["cost_ce"]), _lib.ptr(c["cost_siou"]), _lib.ptr(c["col_sum"]),
                 _lib.ptr(n_valid, i32), n_global, k, _lib.ptr(row_of_col, i32), _lib.ptr(losses))
        fctx.save_for_backward(pred, gt_row, row_of_col, n_valid, c["tp"], c["col_sum"], c["row_count"])
        fctx.in_shape, fctx.n_global = pred_ins.shape, n_global
        fctx.mark_non_differentiable(n_valid, row_of_col)
        return losses[0].clone(), losses[1].clone(), losses[2].clone(), n_valid, row_of_col

    @staticmethod
    def backward(fctx, g_ce, g_inv, g_siou, _g_n=None, _g_r=None):
        d_pred = _loss_backward(fctx.saved_tensors, fctx.n_global, (g_ce, g_inv, g_siou))
        return d_pred.reshape(fctx.in_shape), None, None, None


_STATUS_TEXT = {701: "a label outside [0, 65536)", 702: "more distinct labels than ins_num (or an empty batch)"}


def _check_status(device, what, hint=""):
    """Raise if an earlier device-side call rejected its labels (the error word is read and cleared without synchronising)."""
    code = get_context(device).lib.dmnerf_ins_status_take()
    if code:
        raise RuntimeError("%s: an earlier call was given %s (code %d); its loss was NaN and its gradient zero%s"
                           % (what, _STATUS_TEXT.get(code, "labels it cannot rank"), code, hint))


def ins_assignment(pred_ins, gt_labels, ins_num):
    """Device-side matching only: (row_of_col [ins_num] int32: rank of the matched label per prediction channel or -1,
    n_valid [1] int32), both on the device.  Same kernels as ins_criterion; for tests and diagnostics."""
    labels = gt_labels.to(pred_ins.device).reshape(-1).to(torch.int32).contiguous()
    out = _MatchedLossDevice.apply(pred_ins, labels, pred_ins.shape[0], None)
    return out[4], out[3]


def ins_criterion(pred_ins, gt_labels, ins_num):
    """evaluator.py:19-37.  pred_ins [N, ins_num] (rendered instance probabilities, CUDA), gt_labels [N] (object ids)."""
    if not pred_ins.is_cuda:
        raise RuntimeError("ins_criterion: expected CUDA tensors (no CPU fallback)")
    if pred_ins.dim() != 2 or pred_ins.shape[1] != ins_num or gt_labels.shape[0] != pred_ins.shape[0]:
        raise RuntimeError("ins_criterion: pred_ins %s / gt_labels %s / ins_num %d are inconsistent"
                           % (tuple(pred_ins.shape), tuple(gt_labels.shape), ins_num))
    labels = gt_labels.to(pred_ins.device).reshape(-1)
    if os.environ.get("DMNERF_INS_ASSIGN", "device") != "host":
        _check_status(pred_ins.device, "ins_criterion",
                      ". DMNERF_INS_ASSIGN=host handles arbitrary integer labels (one synchronisation per call).")
        valid_ce, invalid_ce, valid_siou, _, _ = _MatchedLossDevice.apply(pred_ins, labels.to(torch.int32).contiguous(),
                                                                          pred_ins.shape[0], None)
        # evaluator.py:33 returns tensor([0]) (shape [1]) when every channel is matched; here invalid_ce is a 0-dim zero in that
        # case (the number of distinct labels is not known on the host)
        return valid_ce + invalid_ce + valid_siou, valid_ce, invalid_ce, valid_siou             # evaluator.py:36
    try:
        # object ids in [0, ins_num) (every dataset of the reference): the id IS the cost-matrix row; which ids occur comes back
        # with the matrices, so the call makes a single device->host hop (no torch.unique synchronisation)
        valid_ce, invalid_ce, valid_siou, n_valid_t = _MatchedLoss.apply(pred_ins, labels.to(torch.int32).contiguous(), None)
    except _LabelsOutOfRange:
        valid = torch.unique(labels)                                                        # evaluator.py:21 (sorted)
        n_valid = int(valid.numel())
        if n_valid > ins_num:
            raise RuntimeError("ins_criterion: %d distinct labels for ins_num %d" % (n_valid, ins_num))
        gt_row = torch.searchsorted(valid, labels).to(torch.int32).contiguous()             # column of the one-hot, :25
        valid_ce, invalid_ce, valid_siou, n_valid_t = _MatchedLoss.apply(pred_ins, gt_row, n_valid)
    if int(n_valid_t) == ins_num:
        invalid_ce = torch.tensor([0], device=pred_ins.device)                              # evaluator.py:33
    ins_loss_sum = valid_ce + invalid_ce + valid_siou                                       # evaluator.py:36
    return ins_loss_sum, valid_ce, invalid_ce, valid_siou
