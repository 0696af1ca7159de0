"""CPU oracle of moving pieces -- TEST INFRASTRUCTURE ONLY (the product package never imports it).

Restates DESIGN.md, "Moving pieces" on top of the region oracle (region_oracle.lookup / sample_points, fp32 bit for bit) and
the label rule of objects_oracle (argmax of the sigmoid over every instance channel, first maximum):
  piece_vote        per move, vote(r) = in(r) >= out(r), the fine pass's weights of the label's samples inside / outside the
                    piece, each summed in ascending sample order in fp32;
  exchanger_pieces  dmnerf_oracle.exchanger with every `label == mv` replaced by "is the moving piece" (equal to it without
                    pieces, and with an all-ones region that keeps samples outside the grid);
  manipulator       dmnerf_oracle.manipulator, unchanged, with its exchange step replaced by exchanger_pieces: an exchange hook
                    that swaps the module's exchanger for the call and finds each exchanged raw's rays and depths, and the
                    first fine pass of every ray set, among the network calls the pipeline made.
A region here is a dict: vmap float32 [3, 4], bits uint32 words, dim, applies (4 label words), outside_keep (bool)."""
import contextlib

import numpy as np
import torch

from . import dmnerf_oracle as O
from . import region_oracle as RO
from .objects_oracle import object_labels


def region_of(region, ins_num):
    """The oracle dict of an objects.Region (its bits copied to the host)."""
    return {"vmap": np.asarray(region.voxel_map, dtype=np.float32).reshape(3, 4),
            "bits": region.bits.detach().cpu().numpy().view(np.uint32), "dim": int(region.dim),
            "applies": [int(w) & 0xFFFFFFFF for w in region.applies_words(ins_num)], "outside_keep": region.outside == "keep"}


def _np(t, dtype=np.float32):
    return t.detach().cpu().numpy().astype(dtype) if torch.is_tensor(t) else np.asarray(t, dtype=dtype)


def in_piece(region, mv, rays_o, rays_d, z):
    """bool [N, S]: a sample of label mv at p = o + d z (fp32) is in the piece (the region does not drop it)."""
    if not (int(region["applies"][mv >> 5]) >> (mv & 31)) & 1:
        raise ValueError("moved label %d is not among the labels its region applies to" % mv)
    z = _np(z)
    n, s = z.shape
    b = RO.lookup(region["vmap"], region["bits"], region["dim"],
                  RO.sample_points(_np(rays_o), _np(rays_d), z).reshape(-1, 3)).reshape(n, s)
    return ~((b == 0) | ((b < 0) & (not region["outside_keep"])))


def piece_vote(raw, z, weights, rays_o, rays_d, move_labels, regions):
    """uint8 [m, N]: per move i, in >= out, where in (out) = sum of weights over the samples labelled move_labels[i] that the
    region keeps (drops), added one sample at a time from s = 0 in fp32; 1 for a move without a region."""
    labels = object_labels(raw).cpu().numpy()
    w = _np(weights)
    n, s = w.shape
    out = np.ones((len(move_labels), n), dtype=np.uint8)
    zero = np.float32(0)
    for i, (mv, reg) in enumerate(zip(move_labels, regions)):
        if reg is None:
            continue
        mv = int(mv)
        inside = in_piece(reg, mv, rays_o, rays_d, z)
        lab = labels == mv
        acc_in, acc_out = np.zeros(n, dtype=np.float32), np.zeros(n, dtype=np.float32)
        for k in range(s):
            acc_in = acc_in + np.where(lab[:, k] & inside[:, k], w[:, k], zero)
            acc_out = acc_out + np.where(lab[:, k] & ~inside[:, k], w[:, k], zero)
        out[i] = (acc_in >= acc_out).astype(np.uint8)
    return out


def exchanger_pieces(ori_raw, tar_raws, ori_raw_pred, tar_raw_preds, move_labels, pieces=None):
    """The exchange with pieces -> (edited ori_raw, tar_raws, per-sample label of the original, of the last target).
    pieces: None, or a dict with regions (a region dict or None per move), rest_drop (bool per move), ori_rays (o, d), ori_z
    [N, S], tar_rays [(o, d)], tar_zs [[N, S]], ori_votes [m, N] and tar_votes [[N]] (target i's vote for move i)."""
    ori_raw = ori_raw.clone()
    ori_label = torch.argmax(torch.sigmoid(ori_raw[..., 4:]), dim=-1)
    ori_acc = torch.argmax(torch.sigmoid(ori_raw_pred[..., :-1]), dim=-1)[:, None].expand_as(ori_label)
    n, s = ori_label.shape
    ones = torch.ones((n, s), dtype=torch.bool)
    from_acc = torch.zeros((n, s), dtype=torch.bool)
    tar_label = None
    for i, mv in enumerate(move_labels):
        mv = int(mv)
        reg = None if pieces is None else pieces["regions"][i]
        tar_raw = tar_raws[i]
        if reg is None:
            in_o = in_t = vote_o = vote_t = ones
            drop_rest = False
        else:
            in_o = torch.from_numpy(in_piece(reg, mv, pieces["ori_rays"][0], pieces["ori_rays"][1], pieces["ori_z"]))
            in_t = torch.from_numpy(in_piece(reg, mv, pieces["tar_rays"][i][0], pieces["tar_rays"][i][1], pieces["tar_zs"][i]))
            vote_o = torch.as_tensor(_np(pieces["ori_votes"][i], np.uint8) != 0)[:, None].expand(n, s)
            vote_t = torch.as_tensor(_np(pieces["tar_votes"][i], np.uint8) != 0)[:, None].expand(n, s)
            drop_rest = bool(pieces["rest_drop"][i])

        def moving(lab, fa, inside, vote):
            return (lab == mv) & torch.where(fa, vote, inside)
        ori_acc_mv = (ori_acc == mv) & vote_o
        fix = moving(ori_label, from_acc, in_o, vote_o) & ~ori_acc_mv                  # occlusion fix
        ori_label = torch.where(fix, ori_acc, ori_label)
        from_acc = from_acc | fix
        ori_mv = moving(ori_label, from_acc, in_o, vote_o)
        filling = ori_acc_mv & ~ori_mv
        tar_label = torch.argmax(torch.sigmoid(tar_raw[..., 4:]), dim=-1)
        tar_acc = torch.argmax(torch.sigmoid(tar_raw_preds[i][..., :-1]), dim=-1)[:, None].expand_as(tar_label)
        tar_acc_mv = (tar_acc == mv) & vote_t
        fix_t = moving(tar_label, torch.zeros_like(fix), in_t, vote_t) & ~tar_acc_mv
        tar_label = torch.where(fix_t, tar_acc, tar_label)
        tar_mv = moving(tar_label, fix_t, in_t, vote_t)
        take = filling | tar_mv
        wipe = ~take & (ori_mv | ((ori_label == mv) & drop_rest))
        ori_raw = torch.where(take[..., None], tar_raw, ori_raw)
        ori_raw = torch.where(wipe[..., None], ori_raw * 0, ori_raw)
    return ori_raw, tar_raws, ori_label, tar_label


@contextlib.contextmanager
def _exchange_hook(target_labels, regions, rest_drop):
    """dmnerf_oracle's manipulator_nerf recorded and its exchanger replaced by exchanger_pieces for the block."""
    calls = []
    real_nerf, real_exchanger = O.manipulator_nerf, O.exchanger
    state = {"votes": None}

    def nerf(p, rays, z_vals=None, n_samples=None, near=None, far=None):
        raw, z = real_nerf(p, rays, z_vals, n_samples, near, far)
        calls.append((raw, rays, z, z_vals is not None))
        return raw, z

    def find(raw):
        for r, rays, z, _ in reversed(calls):
            if r is raw:
                return rays, z
        raise AssertionError("exchange hook: an exchanged raw that no network call returned")

    def exchanger(ori_raw, tar_raws, ori_raw_pred, tar_raw_preds, move_labels):
        m = len(move_labels)
        if state["votes"] is None:                       # the first exchange: the fine passes so far are ori, target 0, 1, ...
            fine = [c for c in calls if c[3]]
            votes = []
            for k, (raw, rays, z, _) in enumerate(fine[:m + 1]):
                w = O.manipulator_render(raw, z, rays[1])[1]
                moves = (list(move_labels), regions) if k == 0 else ([move_labels[k - 1]], [regions[k - 1]])
                votes.append(piece_vote(raw, z, w, rays[0], rays[1], *moves))
            state["votes"] = (votes[0], [v[0] for v in votes[1:]])
        ori_rays, ori_z = find(ori_raw)
        tars = [find(t) for t in tar_raws[:m]]
        pieces = {"regions": regions, "rest_drop": rest_drop, "ori_rays": ori_rays, "ori_z": ori_z,
                  "tar_rays": [t[0] for t in tars], "tar_zs": [t[1] for t in tars],
                  "ori_votes": state["votes"][0], "tar_votes": state["votes"][1]}
        return exchanger_pieces(ori_raw, tar_raws, ori_raw_pred, tar_raw_preds, move_labels, pieces)
    O.manipulator_nerf, O.exchanger = nerf, exchanger
    try:
        yield
    finally:
        O.manipulator_nerf, O.exchanger = real_nerf, real_exchanger


def manipulator(p_coarse, p_fine, ori_rays, f_tar_rays, n_samples, n_importance, near, far, target_labels, us=None, regions=None,
                rest_drop=None):
    """dmnerf_oracle.manipulator with pieces: regions (a region dict or None per label of target_labels), rest_drop (bool per
    move, default keep).  Without a region it is dmnerf_oracle.manipulator itself."""
    m = len(target_labels)
    regions = [None] * m if regions is None else list(regions)
    if all(r is None for r in regions):
        return O.manipulator(p_coarse, p_fine, ori_rays, f_tar_rays, n_samples, n_importance, near, far, target_labels, us=us)
    rest_drop = [False] * m if rest_drop is None else list(rest_drop)
    with _exchange_hook(target_labels, regions, rest_drop):
        return O.manipulator(p_coarse, p_fine, ori_rays, f_tar_rays, n_samples, n_importance, near, far, target_labels, us=us)
