"""Object manipulation at render time (reference networks/manipulator.py:18-205) on the native kernels: the four functions
of the edit path with the reference's names and signatures.

    exchanger(ori_raw, tar_raws, ori_raw_pred, tar_raw_preds, move_labels)               manipulator.py:18-83   (one kernel)
    manipulator_render(raw, z_vals, rays_d)                                              manipulator.py:86-105  (composite, all instance channels)
    manipulator_nerf(rays, position_embedder, view_embedder, model, N_samples, near, far, z_vals)   manipulator.py:108-134 (tensor-core network)
    manipulator(position_embedder, view_embedder, model_coarse, model_fine, ori_rays, f_tar_rays, args)   manipulator.py:137-205

The two loops that drive it, with the reference's signatures, printed lines and output files (no lpips, skimage, cv2 or imageio):

    manipulator_eval(position_embedder, view_embedder, model_coarse, model_fine, ori_poses, hwk, trans_dicts, save_dir, ins_rgbs,
                     args, gt_rgbs=None, gt_labels=None)                                  manipulator.py:208-364
    manipulator_demo(position_embedder, view_embedder, model_coarse, model_fine, ori_poses, hwk, objs_trans, save_dir, ins_rgbs,
                     objs, view_poses, ins_map, args)                                     manipulator.py:367-491

Both render through manipulate_frame (one edited frame, args.N_test rays per manipulator() call, outputs preallocated on the
device) and keep every per-pixel step on the device: rays, metrics (dmnerf_b200.tester), label arg-max and colours.  The host
reads back the metric result struct and the PNG images once per frame.  Rules and deviations: DESIGN.md, "Manipulation loops".

Each of them also takes the keywords pieces= and rest= (no counterpart in the original; DESIGN.md, "Moving pieces"): a move may
carry a region, so that one piece of its label moves and the rest of the label is kept or dropped.  Without them the edit is the
original's.
"""
import ctypes as C
import json
import os
import time

import numpy as np
import torch

from . import _lib
from .engine import get_context
from .autograd import mlp_forward_rays
from .render import composite, _check_embedders
from .helpers import sample_pdf, sort_concat, get_rays_k


def exchanger(ori_raw, tar_raws, ori_raw_pred, tar_raw_preds, move_labels, pieces=None):
    """Edits `ori_raw` in place like the reference and returns (ori_raw, tar_raws, ori_pred_label, tar_pred_label).
    pieces: an ExchangePieces (DESIGN.md, "Moving pieces"), or None for the reference's exchanger."""
    if not ori_raw.is_cuda:
        raise RuntimeError("exchanger: expected CUDA tensors (no CPU fallback)")
    if not (ori_raw.is_contiguous() and ori_raw.dtype == torch.float32):
        raise RuntimeError("exchanger: ori_raw must be a contiguous float32 tensor (it is edited in place)")
    n, s, c = ori_raw.shape
    m = len(move_labels)
    tars = [t.contiguous().float() for t in tar_raws]
    accs = [a.contiguous().float() for a in tar_raw_preds]
    acc_o = ori_raw_pred.contiguous().float()
    if len(tars) < m or len(accs) < m or any(t.shape != ori_raw.shape for t in tars[:m]) or acc_o.shape != (n, c - 4):
        raise RuntimeError("exchanger: inconsistent shapes")
    ctx = get_context(ori_raw.device)
    ori_label = torch.empty((n, s), device=ori_raw.device, dtype=torch.int64)
    tar_label = torch.empty((n, s), device=ori_raw.device, dtype=torch.int64)
    mv = (C.c_int * m)(*[int(v) for v in move_labels])
    # desc points into the tensors of `alive`, which stay referenced until the call returns
    desc, alive = (None, ()) if pieces is None else pieces.describe(move_labels, n, s, c - 5, ori_raw.device)
    ctx.call("dmnerf_exchanger", _lib.ptr(ori_raw), _lib.ptrs(tars[:m]), _lib.ptr(acc_o), _lib.ptrs(accs[:m]), mv, m, n, s, c,
             _lib.ptr(ori_label, torch.int64), _lib.ptr(tar_label, torch.int64), None if desc is None else C.byref(desc))
    return ori_raw, tar_raws, ori_label, tar_label


# ----------------------------------------------------------------------------------------------------------------- pieces
# DESIGN.md, "Moving pieces": a move may carry a region (objects.Region), so that only the samples of its label inside that piece
# move; the rest of the label is kept or dropped.  Rays are judged by a per-ray vote on their first fine pass.
RESTS = ("keep", "drop")


def move_rests(rest, m):
    """rest ("keep" / "drop", or one of them per move) -> [bool] of m: True where the rest of the label is dropped."""
    rests = [rest] * m if isinstance(rest, str) else list(rest)
    if len(rests) != m or any(r not in RESTS for r in rests):
        raise ValueError("rest must be 'keep' or 'drop', or one of them for each of the %d moves, got %r" % (m, rest))
    return [r == "drop" for r in rests]


def move_pieces(pieces, move_labels, ins_num, device):
    """pieces (None, or a Region or None per move of move_labels) checked -> a list of m Regions / None, or None when no move has
    a region.  ValueError for a wrong length, a region on another device or a moved label outside the region's labels."""
    m = len(move_labels)
    if pieces is None:
        return None
    pieces = list(pieces)
    if len(pieces) != m:
        raise ValueError("pieces: %d entries for %d moved labels" % (len(pieces), m))
    for r, mv in zip(pieces, move_labels):
        if r is not None:
            _piece_region(r, int(mv), ins_num, device)
    return pieces if any(r is not None for r in pieces) else None


def _piece_region(region, mv, ins_num, device):
    """The C struct of one move's region (None: bits NULL)."""
    if region is None:
        return _lib.RegionDesc()
    from .objects import Region
    if not isinstance(region, Region):
        raise ValueError("pieces: each entry must be an objects.Region or None, got %r" % (type(region).__name__,))
    if region.bits.device != torch.device(device):
        raise ValueError("pieces: a region's bits live on %s, the edit on %s" % (region.bits.device, device))
    d = region.abi(ins_num)
    if not (0 <= mv <= ins_num and (d.applies[mv >> 5] >> (mv & 31)) & 1):
        raise ValueError("pieces: moved label %d is not among the labels its region applies to" % mv)
    return d


def piece_vote(raw, z, weights, rays_o, rays_d, move_labels, regions):
    """dmnerf_piece_vote: per move, does a ray's accumulated label stand for the piece?  raw [N,S,C], depths z [N,S], composite
    weights [N,S] and rays [N,3] of one fine pass -> uint8 [m, N] = (weight of mv's samples the region keeps) >= (weight of those
    it drops), each summed in ascending sample order in fp32; 1 for a move without a region."""
    _lib.need_cuda("piece_vote", raw, z, weights, rays_o, rays_d)
    n, s, c = raw.shape
    m = len(move_labels)
    if len(regions) != m or not 1 <= m <= _lib.MAX_MOVES:
        raise ValueError("piece_vote: between 1 and %d moves, one region (or None) each" % _lib.MAX_MOVES)
    raw, z, weights = raw.contiguous().float(), z.contiguous().float(), weights.contiguous().float()
    rays_o, rays_d = rays_o.contiguous().float(), rays_d.contiguous().float()
    if z.shape != (n, s) or weights.shape != (n, s) or rays_o.shape != (n, 3) or rays_d.shape != (n, 3):
        raise RuntimeError("piece_vote: inconsistent shapes")
    descs = (_lib.RegionDesc * m)(*[_piece_region(r, int(mv), c - 5, raw.device) for r, mv in zip(regions, move_labels)])
    votes = torch.empty((m, n), dtype=torch.uint8, device=raw.device)
    get_context(raw.device).call("dmnerf_piece_vote", _lib.ptr(raw), _lib.ptr(z), _lib.ptr(weights), _lib.ptr(rays_o),
                                 _lib.ptr(rays_d), n, s, c, (C.c_int * m)(*[int(v) for v in move_labels]), descs, m,
                                 _lib.ptr(votes, torch.uint8))
    return votes


class ExchangePieces:
    """The pieces of one exchange: regions (a Region or None per move), rest_drop (bool per move), the original's rays (o, d)
    [N,3] and the depths ori_z [N,S] of ori_raw's samples, each target's rays tar_rays[i] = (o, d) and depths tar_zs[i] [N,S],
    and the votes of the first fine pass: ori_votes uint8 [m, N] (piece_vote of the original rays) and tar_votes[i] uint8 [N]
    (target i's vote for move i)."""

    def __init__(self, regions, rest_drop, ori_rays, ori_z, tar_rays, tar_zs, ori_votes, tar_votes):
        self.regions, self.rest_drop = list(regions), list(rest_drop)
        self.ori_rays, self.ori_z, self.tar_rays, self.tar_zs = ori_rays, ori_z, list(tar_rays), list(tar_zs)
        self.ori_votes, self.tar_votes = ori_votes, list(tar_votes)

    def describe(self, move_labels, n, s, ins_num, device):
        """-> (the dmnerf_pieces struct, the tensors it points into, to be kept alive for the call)."""
        m = len(move_labels)
        if len(self.regions) != m or len(self.rest_drop) != m:
            raise ValueError("exchanger: pieces describe %d moves, %d moved labels given" % (len(self.regions), m))
        d = _lib.Pieces()
        keep = []

        def dev(t, shape, dtype=torch.float32):
            _lib.need_cuda("exchanger", t)
            t = t.contiguous().to(dtype)
            if tuple(t.shape) != shape or t.device != torch.device(device):
                raise RuntimeError("exchanger: a pieces tensor has shape %s on %s, expected %s on %s"
                                   % (tuple(t.shape), t.device, shape, device))
            keep.append(t)
            return _lib.ptr(t, dtype).value
        for i, (r, mv) in enumerate(zip(self.regions, move_labels)):
            d.region[i] = _piece_region(r, int(mv), ins_num, device)
            if r is None:
                continue
            d.rest_drop[i] = int(bool(self.rest_drop[i]))
            d.ori_vote[i] = dev(self.ori_votes[i], (n,), torch.uint8)
            d.tar_vote[i] = dev(self.tar_votes[i], (n,), torch.uint8)
            d.tar_rays_o[i] = dev(self.tar_rays[i][0], (n, 3))
            d.tar_rays_d[i] = dev(self.tar_rays[i][1], (n, 3))
            d.tar_z[i] = dev(self.tar_zs[i], (n, s))
        if any(r is not None for r in self.regions):
            d.ori_rays_o, d.ori_rays_d = dev(self.ori_rays[0], (n, 3)), dev(self.ori_rays[1], (n, 3))
            d.ori_z = dev(self.ori_z, (n, s))
        return d, keep


def manipulator_render(raw, z_vals, rays_d):
    rgb, weights, depth, ins, _ = composite(raw, z_vals, rays_d, keep_all_ins=True)
    return rgb, weights, depth, ins


def manipulator_nerf(rays, position_embedder, view_embedder, model, N_samples=None, near=None, far=None, z_vals=None,
                     impl=_lib.IMPL_AUTO):
    _check_embedders(position_embedder, view_embedder)
    rays_o, rays_d = rays
    n = rays_d.shape[0]
    if z_vals is None:
        dev = rays_d.device
        near_, far_ = near * torch.ones(size=(n, 1), device=dev), far * torch.ones(size=(n, 1), device=dev)
        t_vals = torch.linspace(0., 1., steps=N_samples, device=dev)
        z_vals = (near_ * (1. - t_vals) + far_ * t_vals).expand([n, N_samples])       # manipulator.py:117-120
    raw = mlp_forward_rays(model, rays_o, rays_d, z_vals.contiguous(), impl)
    return raw, z_vals


def _ins_num(model):
    return int(model.ins_linear.weight.shape[0]) - 1


def manipulator(position_embedder, view_embedder, model_coarse, model_fine, ori_rays, f_tar_rays, args, us=None,
                impl=_lib.IMPL_AUTO, pieces=None, rest="keep"):
    """manipulator.py:137-205.  `us`: optional list of [N, N_importance] uniforms replacing the torch.rand draws of the
    sample_pdf calls (order: original rays, every target, original rays again) -- used by the parity tests.
    pieces (DESIGN.md, "Moving pieces"): None, or one objects.Region or None per label of args.target_labels: a move with a
    region moves only the samples of its label inside that piece; rest ("keep" / "drop", or one per move) says what becomes of
    the label's other samples.  Without any region the edit is the reference's."""
    N_samples, N_importance, near, far = args.N_samples, args.N_importance, args.near, args.far
    us = list(us) if us is not None else None
    labels = list(args.target_labels)
    drops = move_rests(rest, len(labels))
    regions = move_pieces(pieces, labels, _ins_num(model_fine), ori_rays.device)

    def draw(bins, w):
        return sample_pdf(bins, w, N_importance, u=(us.pop(0) if us is not None else None))

    def nerf(rays, model, z=None):
        return manipulator_nerf(rays, position_embedder, view_embedder, model, N_samples, near, far, z_vals=z, impl=impl)

    def fine_pass(rays, coarse_raw, coarse_z, moves=None):
        _, w, _, _ = manipulator_render(coarse_raw, coarse_z, rays[1])
        mid = .5 * (coarse_z[..., 1:] + coarse_z[..., :-1])
        z_s = draw(mid, w[..., 1:-1])
        z_full = sort_concat(coarse_z, z_s)                                   # sort(cat(.)) as one kernel
        raw_full, _ = nerf(rays, model_fine, z_full)
        _, w_full, _, ins_acc = manipulator_render(raw_full, z_full, rays[1])
        vote = None if moves is None else piece_vote(raw_full, z_full, w_full, rays[0], rays[1], *moves)
        return z_s, ins_acc, vote

    with torch.no_grad():
        ori_raw, ori_z = nerf(ori_rays, model_coarse)
        _, ori_ins_acc, ori_votes = fine_pass(ori_rays, ori_raw, ori_z, None if regions is None else (labels, regions))
        tar_raws, tar_zs, tar_samples, tar_accs, tar_votes = [], [], [], [], []
        tar_rgb = None
        for idx, tar_rays in enumerate(f_tar_rays):
            t_raw, t_z = nerf(tar_rays, model_coarse)
            tar_rgb, _, _, _ = manipulator_render(t_raw, t_z, tar_rays[1])
            moves = None if regions is None or idx >= len(labels) else ([labels[idx]], [regions[idx]])
            z_s, acc, vote = fine_pass(tar_rays, t_raw, t_z, moves)
            tar_raws.append(t_raw); tar_zs.append(t_z); tar_samples.append(z_s); tar_accs.append(acc)
            tar_votes.append(None if vote is None else vote[0])

        def pieces_on(ori_depths, tar_depths):
            if regions is None:
                return None
            return ExchangePieces(regions, drops, ori_rays, ori_depths, f_tar_rays, tar_depths, ori_votes, tar_votes)
        ori_raw, _, _, _ = exchanger(ori_raw, tar_raws, ori_ins_acc, tar_accs, labels, pieces=pieces_on(ori_z, tar_zs))
        _, ori_w, _, _ = manipulator_render(ori_raw, ori_z, ori_rays[1])
        mid = .5 * (ori_z[..., 1:] + ori_z[..., :-1])
        ori_samples = draw(mid, ori_w[..., 1:-1])
        extra = torch.cat([ori_samples] + tar_samples, -1)                     # samples every second-pass ray set shares
        ori_z2 = sort_concat(ori_z, extra)
        ori_raw2, _ = nerf(ori_rays, model_fine, ori_z2)
        tar_z2s = []
        for idx, tar_rays in enumerate(f_tar_rays):
            t_z2 = sort_concat(tar_zs[idx], extra)
            tar_raws[idx], _ = nerf(tar_rays, model_fine, t_z2)
            tar_z2s.append(t_z2)
        ori_raw2, _, _, _ = exchanger(ori_raw2, tar_raws, ori_ins_acc, tar_accs, labels, pieces=pieces_on(ori_z2, tar_z2s))
        final_rgb, _, _, final_ins = manipulator_render(ori_raw2, ori_z2, ori_rays[1])
    return final_rgb, final_ins, tar_rgb, tar_accs[-1]


# ----------------------------------------------------------------------------------------------------------------- frame loops
def manipulate_frame(H, W, K, ori_pose, tar_rays_o, tar_rays_d, position_embedder, view_embedder, model_coarse, model_fine, args,
                     impl=_lib.IMPL_AUTO, pieces=None, rest="keep"):
    """One edited frame (the chunk loops of manipulator.py:246-269 and :445-466): manipulator() over the H*W rays of
    get_rays_k(H, W, K, ori_pose), args.N_test rays per call with the last call partial, targets labelled args.target_labels.
    tar_rays_o / tar_rays_d: [T, H*W, 3] CUDA rays of the T targets.  The sample_pdf draws keep the reference's order (per
    chunk: the original rays, every target, the original rays again), so a run seeded like the reference consumes the default
    CUDA generator identically.  Returns final rgb [H*W, 3], final ins [H*W, ins_num + 1], tar_rgb [H*W, 3] and
    tar_ins_accum [H*W, ins_num + 1] (of the last target), written chunk by chunk into preallocated device tensors.
    pieces / rest: as manipulator() (one Region or None per label of args.target_labels; "keep" / "drop"), checked once here."""
    dev = tar_rays_o.device
    move_rests(rest, len(args.target_labels))
    move_pieces(pieces, list(args.target_labels), _ins_num(model_fine), dev)
    ori_o, ori_d = get_rays_k(H, W, K, torch.as_tensor(ori_pose, dtype=torch.float32, device=dev))
    ori_o, ori_d = ori_o.reshape(-1, 3), ori_d.reshape(-1, 3)
    n, chunk = H * W, int(args.N_test)
    if tuple(tar_rays_o.shape[1:]) != (n, 3) or tar_rays_d.shape != tar_rays_o.shape or tar_rays_o.shape[0] < 1:
        raise ValueError("manipulate_frame: target rays must be [T, %d, 3], got %s and %s"
                         % (n, tuple(tar_rays_o.shape), tuple(tar_rays_d.shape)))
    out = None
    with torch.no_grad():
        for step in range(0, n, chunk):
            end = min(step + chunk, n)
            ori = torch.stack([ori_o[step:end], ori_d[step:end]], 0)
            tar = torch.stack([tar_rays_o[:, step:end], tar_rays_d[:, step:end]], 1)               # [T, 2, cnt, 3]
            maps = manipulator(position_embedder, view_embedder, model_coarse, model_fine, ori, tar, args, impl=impl, pieces=pieces,
                               rest=rest)
            if out is None:
                out = [torch.empty((n,) + tuple(m.shape[1:]), device=dev, dtype=m.dtype) for m in maps]
            for o, m in zip(out, maps):
                o[step:end] = m
    return tuple(out)


# deform_v of manipulator.py:381-382: one x amplitude per demo view of the 'sin' deformation
_DEFORM_V = np.concatenate((np.linspace(0, 0.18, 2), np.linspace(0.18, 0, 2), np.linspace(0, -0.18, 2), np.linspace(-0.18, 0, 2)))
DEFORM_FUNCS = ("sin", "ex", "linear", "abs_linear", "ln")


def deform_offsets(deform_func, H, view):
    """Per-row x offsets [H] float64 of a deformed object in demo view `view`, with the numpy expressions of
    manipulator.py:398-426 (the reference repeats each row's value over the W columns)."""
    v_1 = np.linspace(1, H, H)
    if deform_func == 'sin':
        if not 0 <= view < len(_DEFORM_V):
            raise ValueError("manipulator_demo: the 'sin' deformation has amplitudes for %d views, view %d asked"
                             % (len(_DEFORM_V), view))
        return np.sin(((8 * np.pi) / 400) * v_1) * _DEFORM_V[view]
    if deform_func == 'ex':
        return np.exp(-1 * v_1 / 50)
    if deform_func == 'linear':
        return (v_1 - 200) / 215
    if deform_func == 'abs_linear':
        return np.abs(v_1 - 200) / 200
    if deform_func == 'ln':
        return np.log(v_1 / 200)
    raise ValueError("manipulator_demo: unknown deform_func %r (one of %s)" % (deform_func, ", ".join(DEFORM_FUNCS)))


def deformed_rays(ori_o, ori_d, offsets, H, W):
    """Target rays of a deformed object (manipulator.py:427-429): origins [H*W, 3] shifted in x by the row's float64 offset, the
    sum taken in float64 and rounded once to float32 like the reference's fp32 + fp64 tensor add; directions unchanged."""
    off = torch.as_tensor(np.ascontiguousarray(offsets, dtype=np.float64)).to(ori_o.device)
    tar_o = ori_o.clone()
    x = tar_o.view(H, W, 3)[..., 0]
    x.copy_(x.double() + off[:, None])
    return tar_o, ori_d.clone()


def rigid_rays(H, W, K, trans, pose):
    """Target rays of a moved object: get_rays_k(trans @ pose), the product taken with torch in float32 on pose's device."""
    t = torch.as_tensor(np.asarray(trans, dtype=np.float32) if not torch.is_tensor(trans) else trans, dtype=torch.float32,
                        device=pose.device)
    o, d = get_rays_k(H, W, K, t @ pose)
    return o.reshape(-1, 3), d.reshape(-1, 3)


def _models_device(args, model_fine, who):
    dev = torch.device(getattr(args, "device", None) or next(model_fine.parameters()).device)
    if dev.type != "cuda":
        raise RuntimeError("%s: the models must be on a CUDA device (no CPU fallback)" % who)
    return dev


def _color_dict(args):
    data_info = args.datadir.split('/')
    with open('./data/color_dict.json', 'r') as fh:
        return json.load(fh)[data_info[2]][data_info[-1]]


def _u8(rgb):
    """to8b (evaluator.py:14) on the device, copied to the host: (255 * clip(x, 0, 1)).astype(uint8)."""
    return (255 * torch.clamp(rgb, 0, 1)).to(torch.uint8).cpu().numpy()


def manipulator_eval(position_embedder, view_embedder, model_coarse, model_fine, ori_poses, hwk, trans_dicts, save_dir, ins_rgbs,
                     args, gt_rgbs=None, gt_labels=None, pieces=None, rest="keep"):
    """networks/manipulator.py manipulator_eval: object args.target_label moved by trans_dicts['transformations'][0] in every
    view of ori_poses.  pieces / rest: as manipulate_frame (a list of one Region or None; DESIGN.md, "Moving pieces").  Files in save_dir/<mode>/: {i}_rgb.png, {i}_ins.png, {i}_rgb_gt.png, {i}_ins_gt.png (the two label
    images in the channel order cv2.imwrite stores), matching_log.json and test_results.txt (PSNR SSIM LPIPS AP50..AP95 per
    frame, then the mean row).  Poses may be numpy arrays, CPU or CUDA tensors; gt_labels any integer type (test_dmsr.py passes
    int8).  With gt_rgbs=None only {i}_rgb.png is written."""
    from . import tester as T
    from .mesh import argmax_rows
    H, W, K = hwk
    H, W = int(H), int(W)
    dev = _models_device(args, model_fine, "manipulator_eval")
    ins_num = int(args.ins_num)
    color_dict = _color_dict(args)
    have_gt = gt_rgbs is not None
    if have_gt:
        gt_img_dev = torch.as_tensor(gt_rgbs).to(dev, torch.float32).contiguous()
        lab_cpu = torch.as_tensor(gt_labels).cpu()
        if lab_cpu.numel() and (int(lab_cpu.min()) < 0 or int(lab_cpu.max()) >= T._MAX_LABEL):
            raise ValueError("manipulator_eval: gt labels must be integers in [0, %d)" % T._MAX_LABEL)
        lab_dev = lab_cpu.to(torch.int32).to(dev).reshape(lab_cpu.shape[0], -1).contiguous()
        gt_lut = T.gt_label_lut(ins_rgbs, color_dict, int(lab_cpu.max()) + 1 if lab_cpu.numel() else 1)[:, ::-1]   # cv2: BGR
        lpips_vgg = T._lpips_model(dev)
        gt_row = torch.empty(H * W, device=dev, dtype=torch.int32)
        n_valid = torch.empty(1, device=dev, dtype=torch.int32)
    trans_dict = trans_dicts['transformations'][0]
    trans = trans_dict['transformation']
    save_dir = os.path.join(save_dir, trans_dict["mode"])
    os.makedirs(save_dir, exist_ok=True)
    args.target_labels = [args.target_label]
    full_map, psnrs, ssims, lpipses, aps = {}, [], [], [], []

    with torch.no_grad():
        for i, ori_pose in enumerate(ori_poses):
            pose = torch.as_tensor(ori_pose, dtype=torch.float32, device=dev)
            tar_o, tar_d = rigid_rays(H, W, K, trans, pose)
            rgb, ins, _, _ = manipulate_frame(H, W, K, pose, tar_o[None], tar_d[None], position_embedder, view_embedder, model_coarse,
                                              model_fine, args, pieces=pieces, rest=rest)
            rgb = rgb.reshape(H, W, 3).contiguous()
            ins_map = {}
            if have_gt:
                print('=' * 50, i, '=' * 50)
                valid_gt = torch.unique(lab_cpu[i])
                psnr_i, ssim_i, lpips_i, ap, ins_map, _ = T._frame_metrics(
                    "manipulator_eval", i, rgb, gt_img_dev[i], ins[:, :ins_num].contiguous(), lab_dev[i], valid_gt, ins_num,
                    lpips_vgg, gt_row, n_valid)
                psnrs.append(psnr_i)
                ssims.append(ssim_i)
                lpipses.append(lpips_i)
                full_map[i] = ins_map
                aps.append(ap)

            T.write_png(os.path.join(save_dir, f'{i}_rgb.png'), _u8(rgb))
            if have_gt:
                label = argmax_rows(ins).reshape(H, W)                           # all ins_num + 1 channels
                lut = T.pred_label_lut(ins_map, ins_rgbs, color_dict, ins.shape[1])[:, ::-1]
                T.write_png(os.path.join(save_dir, f'{i}_ins.png'), T.colorize(label, lut).cpu().numpy())
                T.write_png(os.path.join(save_dir, f'{i}_rgb_gt.png'), _u8(gt_img_dev[i]))
                T.write_png(os.path.join(save_dir, f'{i}_ins_gt.png'), T.colorize(lab_dev[i].reshape(H, W), gt_lut).cpu().numpy())

    if have_gt:
        with open(os.path.join(save_dir, 'matching_log.json'), 'w') as f:
            json.dump(full_map, f)
        aps = np.array(aps)
        output = np.stack([psnrs, ssims, lpipses, aps[:, 0], aps[:, 1], aps[:, 2], aps[:, 3], aps[:, 4], aps[:, 5]])
        output = output.transpose([1, 0])
        out_ap = np.mean(aps, axis=0)
        mean_output = np.array([np.nanmean(psnrs), np.nanmean(ssims), np.nanmean(lpipses), out_ap[0],
                                out_ap[1], out_ap[2], out_ap[3], out_ap[4], out_ap[5]]).reshape([1, 9])
        output = np.concatenate([output, mean_output], 0)
        np.savetxt(fname=os.path.join(save_dir, 'test_results.txt'), X=output, fmt='%.6f', delimiter=' ')
        print('=' * 49, 'Avg', '=' * 49)
        print('PSNR: {:.4f}, SSIM: {:.4f},  LPIPS: {:.4f} '.format(np.mean(psnrs), np.mean(ssims), np.mean(lpipses)))
        print('AP50: {:.4f}, AP75: {:.4f}, AP80: {:.4f}, AP85: {:.4f}, AP90: {:.4f}, AP95: {:.4f}'
              .format(out_ap[0], out_ap[1], out_ap[2], out_ap[3], out_ap[4], out_ap[5]))


def manipulator_demo(position_embedder, view_embedder, model_coarse, model_fine, ori_poses, hwk, objs_trans, save_dir, ins_rgbs,
                     objs, view_poses, ins_map, args, pieces=None, rest="keep"):
    """networks/manipulator.py manipulator_demo: every object of `objs` edited at once in every view of view_poses (ori_poses
    is unused, as in the reference).  pieces / rest: as manipulate_frame, aligned with `objs` (DESIGN.md, "Moving pieces").  Rigid objects move by objs_trans[obj_name][i]['transformation']; deformed ones shift
    the origins of the view's rays in x (deform_func sin / ex / linear / abs_linear / ln).  Files in save_dir/<args.mani_type>/:
    {i}_rgb.png, {i}_ins.png (label colours through ins_map, cv2's channel order) and {i}_ins_pred_mask.png (the labels as
    uint8); prints `Image{i}: <seconds>` per view."""
    from . import tester as T
    from .mesh import argmax_rows
    H, W, K = hwk
    H, W = int(H), int(W)
    dev = _models_device(args, model_fine, "manipulator_demo")
    color_dict = _color_dict(args)
    save_dir = os.path.join(save_dir, args.mani_type)
    os.makedirs(save_dir, exist_ok=True)
    lut = T.pred_label_lut(ins_map, ins_rgbs, color_dict, int(args.ins_num) + 1)[:, ::-1]

    with torch.no_grad():
        for i, view_pose in enumerate(view_poses):
            time_0 = time.time()
            pose = torch.as_tensor(view_pose, dtype=torch.float32, device=dev)
            ori_o = ori_d = None
            tar_os, tar_ds, target_labels = [], [], []
            for obj in objs:
                target_labels.append(obj['tar_id'])
                if obj['mani_mode'] == 'deform':
                    if ori_o is None:
                        ori_o, ori_d = (r.reshape(-1, 3) for r in get_rays_k(H, W, K, pose))
                    o, d = deformed_rays(ori_o, ori_d, deform_offsets(obj['deform_func'], H, i), H, W)
                else:
                    o, d = rigid_rays(H, W, K, objs_trans[obj['obj_name']][i]['transformation'], pose)
                tar_os.append(o)
                tar_ds.append(d)
            args.target_labels = target_labels
            rgb, ins, _, _ = manipulate_frame(H, W, K, pose, torch.stack(tar_os), torch.stack(tar_ds), position_embedder,
                                              view_embedder, model_coarse, model_fine, args, pieces=pieces, rest=rest)
            label = argmax_rows(ins).reshape(H, W)
            T.write_png(os.path.join(save_dir, f'{i}_rgb.png'), _u8(rgb.reshape(H, W, 3)))
            T.write_png(os.path.join(save_dir, f'{i}_ins.png'), T.colorize(label, lut).cpu().numpy())
            T.write_png(os.path.join(save_dir, f'{i}_ins_pred_mask.png'), label.to(torch.uint8).cpu().numpy())
            time_1 = time.time()
            print(f"Image{i}: {time_1 - time_0}")
