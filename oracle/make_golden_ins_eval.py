"""Generate tests/golden/ins_eval.npz from the UNMODIFIED original ins_eval (networks/evaluator.py:125-175), called the way
render_test calls it (networks/tester.py:97-118), and pin the oracle (oracle/metrics.py) to it.

Each case is checked to be decidable by any correct implementation: its optimal assignment is unique (in the matched predicted
label of every gt object) by a cost margin > 1e-5, and the confidences of its matched predictions have no ties.  Otherwise the
original's fp32 summation order or its non-stable sort would decide the result.

    python oracle/make_golden_ins_eval.py
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFERENCE = os.environ.get("DMNERF_REFERENCE_ROOT", "/root/reference")
sys.path.insert(0, ROOT)
sys.path.insert(0, REFERENCE)
from networks.evaluator import ins_eval as ref_ins_eval      # noqa: E402
from oracle import metrics as M                               # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
Q = 65536                                                     # instance maps are stored as uint16 numerators: value = q / Q


def make_case(rng, H, W, ins_num, n_gt, n_channels, unlabelled=None):
    """gt: Voronoi regions with arbitrary object ids; prediction: each gt object drawn on one of n_channels channels (several
    objects share a channel when n_channels < n_gt), 10% of the pixels on a random channel, two small distractor values."""
    ids = np.sort(rng.choice(np.arange(ins_num), n_gt, replace=False))
    seeds = rng.uniform(0, 1, (n_gt, 2)) * [H, W]
    yy, xx = np.mgrid[0:H, 0:W]
    d = (yy[..., None] - seeds[:, 0]) ** 2 + (xx[..., None] - seeds[:, 1]) ** 2
    region = np.argmin(d, -1)
    gt = ids[region]
    if unlabelled is not None:                                # ScanNet-style crop: some pixels carry an id >= ins_num
        gt = np.where(rng.uniform(size=(H, W)) < 0.08, unlabelled, gt)
    chans = rng.permutation(ins_num)[:n_channels]
    chan_of_obj = chans[rng.integers(0, n_channels, n_gt)] if n_channels < n_gt else chans[rng.permutation(n_gt) % n_channels]
    hot = chan_of_obj[region]
    noise = rng.uniform(size=(H, W)) < 0.10
    # fewer channels than objects: the noise stays on those channels, so some columns of the assignment are empty
    hot = np.where(noise, rng.choice(chans, (H, W)) if n_channels < n_gt else rng.integers(0, ins_num, (H, W)), hot)
    q = np.zeros((H, W, ins_num), np.uint16)
    q_main = rng.integers(Q // 3, Q - 1, (H, W))
    for _ in range(2):
        c = rng.integers(0, ins_num, (H, W))
        np.put_along_axis(q, c[..., None], rng.integers(1, Q // 4, (H, W, 1)).astype(np.uint16), -1)
    np.put_along_axis(q, hot[..., None], q_main[..., None].astype(np.uint16), -1)
    return q, gt.astype(np.int64)


def run_reference(pred, gt_label, ins_num, crop):
    """tester.py:97-118 around the original ins_eval."""
    gt_label = torch.from_numpy(gt_label)
    H, W = gt_label.shape
    gt_ins = torch.zeros(size=(H, W, ins_num))
    valid_gt_labels = torch.unique(gt_label)
    if crop:
        valid_gt_labels = valid_gt_labels[:-1]
    gt_num = len(valid_gt_labels)
    gt_ins[..., :gt_num] = F.one_hot(gt_label.long())[..., valid_gt_labels.long()].float()
    mask = (gt_label < ins_num).type(torch.float32) if crop else None
    pred_label, ap, ret = ref_ins_eval(torch.from_numpy(pred), gt_ins, gt_num, ins_num, mask)
    return pred_label.numpy(), np.array(ap, np.float64), np.asarray(ret, np.int64), valid_gt_labels.numpy(), gt_num


def gt_ranks(gt_label, valid):
    rank = np.searchsorted(valid, gt_label)
    ok = (rank < len(valid)) & (valid[np.minimum(rank, len(valid) - 1)] == gt_label)
    return np.where(ok, rank, -1).astype(np.int32)


CASES = [
    # tag, H, W, ins_num, gt objects, predicted channels, unlabelled id (crop path) or None
    ("k13", 48, 64, 13, 9, 9, None),
    ("k59_crop", 40, 56, 59, 20, 20, 255),
    ("k93", 96, 128, 93, 40, 40, None),
    ("more_gt", 48, 64, 13, 10, 6, None),                 # gt objects matched to empty columns
    ("empty_cols", 32, 40, 13, 12, 4, None),              # several identical empty columns: scipy's tie rule decides
]


def main():
    save = {}
    for ci, (tag, H, W, ins_num, n_gt, n_ch, unl) in enumerate(CASES):
        rng = np.random.default_rng(1000 + ci)
        for attempt in range(50):
            q, gt = make_case(rng, H, W, ins_num, n_gt, n_ch, unl)
            pred = (q.astype(np.float32) / np.float32(Q)).astype(np.float32)
            crop = unl is not None
            pl, ap, ret, valid, gt_num = run_reference(pred, gt, ins_num, crop)
            rows = gt_ranks(gt, valid)
            masked = (gt >= ins_num).reshape(-1) if crop else None
            o = M.ins_eval(pred.reshape(-1, ins_num), rows.reshape(-1), gt_num, ins_num, masked)
            nv = len(o["valid"])
            margin = M.assignment_margin((o["cost_ce"] + o["cost_siou"])[:gt_num], o["col_of_row"], nv)
            conf = o["median"][o["col_of_row"][o["col_of_row"] < nv]]
            if margin > 1e-5 and len(np.unique(conf)) == len(conf) and (conf > 0).all():
                break
        else:
            raise SystemExit("case %s: no decidable frame in 50 draws" % tag)
        assert np.array_equal(o["pred_label"], pl.reshape(-1)), "oracle pred_label != original (%s)" % tag
        assert np.array_equal(o["return_labels"], ret), "oracle return_labels != original (%s): %s vs %s" % (tag, o["return_labels"], ret)
        assert np.allclose(o["ap"], ap, rtol=0, atol=1e-6), "oracle AP != original (%s): %s vs %s" % (tag, o["ap"], ap)
        save.update({"q_" + tag: q, "gt_" + tag: gt.astype(np.int32), "ins_num_" + tag: ins_num, "crop_" + tag: int(crop),
                     "pred_label_" + tag: pl.astype(np.int64), "ap_" + tag: ap, "return_labels_" + tag: ret,
                     "valid_gt_" + tag: valid.astype(np.int64)})
        print("case %-10s %dx%d ins_num %d: %d gt, %d predicted labels, margin %.3g, AP %s, matched %s"
              % (tag, H, W, ins_num, gt_num, nv, margin, np.round(ap, 4).tolist(), ret.tolist()))
    save["tags"] = np.array([c[0] for c in CASES])
    save["Q"] = Q
    np.savez_compressed(os.path.join(OUT, "ins_eval.npz"), **save)
    print("written", os.path.join(OUT, "ins_eval.npz"), os.path.getsize(os.path.join(OUT, "ins_eval.npz")) // 1024, "KB")


if __name__ == "__main__":
    main()
