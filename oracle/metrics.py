"""CPU checker of the test-view metrics (numpy / scipy): PSNR and SSIM restated from scikit-image 0.18.3, and ins_eval +
calculate_ap (networks/evaluator.py:77-175, integral method) restated through the joint histogram of the two label maps.

The one intended difference from the original: matches are ordered by confidence with a STABLE sort (ties keep gt order); the
original's torch.argsort(descending=True) is not stable."""
import numpy as np
from scipy.ndimage import uniform_filter
from scipy.optimize import linear_sum_assignment

THRESHOLDS = np.array([0.5, 0.75, 0.8, 0.85, 0.9, 0.95], dtype=np.float32)     # compared in fp32, as torch does
CE_TERM = np.float32(-np.log(np.float32(1e-8)))                                 # -log(0 + 1e-8) of one mismatched pixel


def psnr(rgb, gt):
    """peak_signal_noise_ratio(rgb, gt, data_range=1): fp32 difference and square, fp64 mean."""
    d = np.asarray(rgb, np.float32) - np.asarray(gt, np.float32)
    mse = np.mean(d * d, dtype=np.float64)
    with np.errstate(divide="ignore"):
        return float(10 * np.log10(1.0 / mse))


def ssim(rgb, gt):
    """structural_similarity(rgb, gt, multichannel=True, data_range=1)."""
    x, y = np.asarray(rgb), np.asarray(gt)
    if x.shape[0] < 7 or x.shape[1] < 7:
        raise ValueError("win_size exceeds image extent")
    out = []
    for ch in range(x.shape[-1]):
        a, b = x[..., ch].astype(np.float64), y[..., ch].astype(np.float64)
        f = lambda v: uniform_filter(v, size=7)
        ux, uy, uxx, uyy, uxy = f(a), f(b), f(a * a), f(b * b), f(a * b)
        cov_norm = 49 / 48
        vx, vy, vxy = cov_norm * (uxx - ux * ux), cov_norm * (uyy - uy * uy), cov_norm * (uxy - ux * uy)
        C1, C2 = 0.01 ** 2, 0.03 ** 2
        S = ((2 * ux * uy + C1) * (2 * vxy + C2)) / ((ux ** 2 + uy ** 2 + C1) * (vx + vy + C2))
        out.append(S[3:-3, 3:-3].mean())
    return float(np.mean(out))


def calculate_ap(ious, gt_number, confidence=None):
    """Integral AP per threshold in fp32, matches ordered by confidence (stable) or by IoU (descending)."""
    ious = np.asarray(ious, np.float32)
    key = ious if confidence is None else np.asarray(confidence, np.float32)
    order = np.argsort(-key, kind="stable")
    vals = ious[order]
    aps = []
    for t in THRESHOLDS:
        tp = np.cumsum(vals > t)
        prec = (tp / np.arange(1, len(tp) + 1)).astype(np.float32)
        rec = tp.astype(np.float32) / np.float32(gt_number)
        mrec = np.concatenate([[0], rec, [1]]).astype(np.float32)
        mprec = np.concatenate([[0], prec, [0]]).astype(np.float32)
        for i in range(len(mprec) - 1, 0, -1):
            mprec[i - 1] = max(mprec[i - 1], mprec[i])
        ap = np.float32(0)
        for i in range(len(mrec) - 1):
            if mrec[i + 1] != mrec[i]:
                ap = np.float32(ap + np.float32((mrec[i + 1] - mrec[i]) * mprec[i + 1]))
        aps.append(float(ap))
    return aps


def ins_eval(pred_ins, gt_row, gt_num, ins_num, masked=None):
    """pred_ins [N, K] float32; gt_row [N] gt rank (anything outside [0, gt_num): no gt object); masked [N] bool or None.
    Returns dict(pred_label, ap, return_labels, valid, median, cost_ce, cost_siou, col_of_row)."""
    pred = np.asarray(pred_ins, np.float32).reshape(-1, ins_num)
    n, k = pred.shape
    label = np.argmax(pred, -1)
    conf = pred.max(-1)
    if masked is not None:
        label = np.where(np.asarray(masked).reshape(-1), k, label)
    present = np.unique(label)
    valid = present[:-1] if masked is not None else present
    valid = valid[valid < k]
    g = np.asarray(gt_row).reshape(-1).astype(np.int64)
    g = np.where((g >= 0) & (g < gt_num), g, gt_num)
    hist = np.zeros((gt_num + 1, k + 1), np.int64)
    np.add.at(hist, (g, label), 1)
    nv = len(valid)
    tp = np.zeros((gt_num, k), np.int64)
    cp = np.zeros(k, np.int64)
    tp[:, :nv] = hist[:gt_num, valid]
    cp[:nv] = hist[:, valid].sum(0)
    cg = hist[:gt_num].sum(1)
    mism = cg[:, None] + cp[None, :] - 2 * tp
    cost_ce = (np.float64(CE_TERM) * mism / n).astype(np.float32)
    tpf, cpf, cgf = tp.astype(np.float32), cp.astype(np.float32)[None, :], cg.astype(np.float32)[:, None]
    den = ((tpf + (cpf - tpf)) + (cgf - tpf)) + np.float32(1e-6)
    cost_siou = (np.float32(1) - tpf / den).astype(np.float32)
    median = np.zeros(k, np.float32)
    for c, lab in enumerate(valid):
        median[c] = np.median(conf[label == lab])
    result = dict(pred_label=label, valid=valid, median=median, cost_ce=cost_ce, cost_siou=cost_siou)
    if gt_num == 0:
        result.update(ap=[1.0] * 6, return_labels=np.zeros(0, np.int64), col_of_row=np.zeros(0, np.int64))
        return result
    rows, cols = linear_sum_assignment((cost_ce + cost_siou)[:gt_num].astype(np.float64))
    col_of_row = np.empty(gt_num, np.int64)
    col_of_row[rows] = cols
    ious = np.float32(1) - cost_siou[np.arange(gt_num), col_of_row]
    hit = col_of_row < nv
    confidence = np.zeros(gt_num, np.float32)
    confidence[hit] = median[col_of_row[hit]]
    return_labels = np.full(gt_num, -1, np.int64)
    return_labels[hit] = valid[col_of_row[hit]]
    result.update(ap=calculate_ap(ious, gt_num, confidence), return_labels=return_labels, col_of_row=col_of_row)
    return result


def assignment_margin(cost, col_of_row, n_valid_cols):
    """Smallest extra cost of any assignment that differs from col_of_row in the matched predicted label of some gt row (empty
    columns, index >= n_valid_cols, count as one label).  > 0 means the optimum is unique in everything ins_eval reports."""
    cost = np.asarray(cost, np.float64)
    gt_num = cost.shape[0]
    best = cost[np.arange(gt_num), col_of_row].sum()
    margin = np.inf
    for g in range(gt_num):
        c = cost.copy()
        if col_of_row[g] < n_valid_cols:
            c[g, col_of_row[g]] = 1e9
        else:
            c[g, n_valid_cols:] = 1e9
        r, cc = linear_sum_assignment(c)
        margin = min(margin, c[r, cc].sum() - best)
    return margin
