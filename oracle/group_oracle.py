"""CPU oracle of moving objects together -- TEST INFRASTRUCTURE ONLY (the product package never imports it).

Restates DESIGN.md, "Moving objects together" in numpy on top of the edit-sweep, arrangement, collision, placement, moved-render and
copy oracles.  A group move is a move dict with "group": the labels G it carries (holding its "label"), and optionally
"applies": the labels its piece applies to (None: every label).  Each rule is the single move's rule with "label == mv" replaced
by "label in G":
  take     in box && label(t) in G && (occ(t) > level || occ_p <= level) && (no piece || keeps(t, label(t))): (o, l) <- (occ(t),
           label(t)) -- the target's own label;
  vacate   (not for a copy) otherwise label_p in G && occ_p > level && (keeps(p, label_p) || rest_drop)  (the render: no level
           test, the box bound instead);
where keeps(x, l) is the piece's test for a label it applies to and True for any other label.  A move without "group" is the
existing move, and delegates to copy_oracle."""
import numpy as np
import torch

from oracle import arrange_oracle as A
from oracle import collide_oracle as CO
from oracle import copy_oracle as CP
from oracle import edit_sweep_oracle as E
from oracle import placement_turn_oracle as TO
from oracle import render_moves_oracle as RM

N_LABELS = A.N_LABELS


def group_of(move):
    return np.asarray(sorted(set(move.get("group") or [move["label"]])), dtype=np.int64)


def keeps(move, pts, lab):
    """The piece's decision at points pts [n, 3] for their labels lab [n]: True without a piece and for a label it does not apply to."""
    piece = move.get("piece")
    if piece is None:
        return np.ones(len(lab), dtype=bool)
    applies = move.get("applies")
    cut = np.ones(len(lab), dtype=bool) if applies is None else np.isin(lab, list(applies))
    return piece.keeps(pts) | ~cut


def take_mask(o, pts, inv, b, move, evaluate, level):
    """The take decisions of one group move on flat state occupancies o [n] at points pts [n, 3] -> (take [n] bool, occ_t [n]
    float32, label_t [n] int64, evaluated)."""
    G = group_of(move)
    lev = np.float32(level)
    t = E.targets(np.asarray(move["trans"], dtype=np.float64)[:3], pts)
    idx = np.nonzero(E.in_box(E.index_of(inv, b, t), move["box"]))[0]
    take = np.zeros(o.shape[0], dtype=bool)
    occ_t = np.zeros(o.shape[0], dtype=np.float32)
    lab_t = np.zeros(o.shape[0], dtype=np.int64)
    if idx.size:
        o_t, l_t = evaluate(t[idx])
        l_t = np.asarray(l_t, dtype=np.int64)
        occ_t[idx], lab_t[idx] = o_t, l_t
        take[idx] = np.isin(l_t, G) & ((np.asarray(o_t) > lev) | (o[idx] <= lev)) & keeps(move, t[idx], l_t)
    return take, occ_t, lab_t, int(idx.size)


def vacate_mask(o, lab, pts, move, level, take):
    if move.get("copy"):
        return np.zeros(o.shape[0], dtype=bool)
    return ~take & np.isin(lab, group_of(move)) & (o > np.float32(level)) & (keeps(move, pts, lab) |
                                                                            bool(move.get("rest_drop", False)))


def apply(o, lab, pts, inv, b, move, evaluate, level):
    """One move on flat grids (edited in place) -> targets evaluated."""
    if "group" not in move:
        return CP.apply(o, lab, pts, inv, b, move, evaluate, level)
    take, occ_t, lab_t, n = take_mask(o, pts, inv, b, move, evaluate, level)
    vacate = vacate_mask(o, lab, pts, move, level, take)
    o[take], lab[take] = occ_t[take], lab_t[take]
    o[vacate] = 0.0
    return n


def edit(occ, labels, T, extents, moves, evaluate, level):
    """edit_sweep_oracle.edit with groups -> (occ, labels, evaluated)."""
    dim = occ.shape[0]
    o, lab = occ.reshape(-1).astype(np.float32).copy(), labels.reshape(-1).astype(np.int64).copy()
    pts = E.sweep_points(T, extents, dim)
    inv, b = E.grid_index_map(T, extents, dim)
    n = sum(apply(o, lab, pts, inv, b, mv, evaluate, level) for mv in moves)
    return o.reshape(occ.shape), lab.reshape(occ.shape).astype(labels.dtype), n


def grid_edit(src_occ, src_labels, occ, labels, T, extents, moves, level):
    """arrange_oracle.grid_edit with groups -> (occ, labels, landed int64 [n], overwritten int64 [n, 128]): overwritten counts
    the solid state points a take lands on that the move does not vacate (for a copy: every one)."""
    landed = np.zeros(len(moves), dtype=np.int64)
    overwritten = np.zeros((len(moves), N_LABELS), dtype=np.int64)
    state_o, state_l = occ.copy(), labels.copy()
    dim = occ.shape[0]
    pts = E.sweep_points(T, extents, dim)
    inv, b = E.grid_index_map(T, extents, dim)
    ev = A.nearest_evaluate(src_occ.astype(np.float32), src_labels.astype(np.int64), inv, b)
    lev = np.float32(level)
    for i, mv in enumerate(moves):
        if "group" not in mv:
            state_o, state_l, land, over = CP.grid_edit(src_occ, src_labels, state_o, state_l, T, extents, [mv], level)
            landed[i], overwritten[i] = land[0], over[0]
            continue
        o, lab = state_o.reshape(-1).astype(np.float32).copy(), state_l.reshape(-1).astype(np.int64).copy()
        take, occ_t, lab_t, _ = take_mask(o, pts, inv, b, mv, ev, level)
        solid_take = take & (occ_t > lev)
        landed[i] = int(solid_take.sum())
        vacated = np.zeros_like(take) if mv.get("copy") else (np.isin(lab, group_of(mv)) &
                                                              (keeps(mv, pts, lab) | bool(mv.get("rest_drop", False))))
        overwritten[i] = np.bincount(lab[solid_take & (o > lev) & ~vacated], minlength=N_LABELS)
        vacate = vacate_mask(o, lab, pts, mv, level, take)
        o[take], lab[take] = occ_t[take], lab_t[take]
        o[vacate] = 0.0
        state_o, state_l = o.reshape(occ.shape), lab.reshape(occ.shape).astype(labels.dtype)
    return state_o, state_l, landed, overwritten


def moved_object(occ, labels, T, extents, move, level):
    """S, bool [dim]^3 in grid order: the grid points p whose target's nearest index is in the box and holds a solid point of a
    label of the group that the piece keeps (placement_turn_oracle.moved_object with the set test)."""
    dim = occ.shape[0]
    o, lab = occ.reshape(-1).astype(np.float32), labels.reshape(-1).astype(np.int64)
    pts = E.sweep_points(T, extents, dim)
    inv, b = E.grid_index_map(T, extents, dim)
    t = E.targets(np.asarray(move["trans"], dtype=np.float64)[:3], pts)
    u = E.index_of(inv, b, t)
    src = E.in_box(u, move["box"])
    q = np.rint(u[src]).astype(np.int64)
    qi = (q[:, 0] * dim + q[:, 1]) * dim + q[:, 2]
    ok = np.isin(lab[qi], group_of(move)) & (o[qi] > np.float32(level)) & keeps(move, t[src], lab[qi])
    src[np.nonzero(src)[0]] = ok
    return src.reshape(occ.shape)


def vacated(occ, labels, T, extents, move, level):
    """The solid points a group move vacates, bool [dim]^3 (none for a copy)."""
    dim = occ.shape[0]
    o, lab = occ.reshape(-1).astype(np.float32), labels.reshape(-1).astype(np.int64)
    pts = E.sweep_points(T, extents, dim)
    out = vacate_mask(o, lab, pts, move, level, np.zeros(o.shape[0], dtype=bool))
    return out.reshape(occ.shape)


def move_overlap(occ, labels, T, extents, moves, level, obstacles=None):
    """collide_oracle.move_overlap with groups (each candidate on its own) -> (overlap int64 [n, 128], landed int64 [n])."""
    overlap = np.zeros((len(moves), N_LABELS), dtype=np.int64)
    landed = np.zeros(len(moves), dtype=np.int64)
    lab = labels.reshape(-1).astype(np.int64)
    is_obst = np.ones(N_LABELS, dtype=bool) if obstacles is None else np.isin(np.arange(N_LABELS), list(obstacles))
    blocking = (occ.reshape(-1) > np.float32(level)) & is_obst[np.clip(lab, 0, N_LABELS - 1)]
    for i, mv in enumerate(moves):
        if "group" not in mv:
            over, land = CP.move_overlap(occ, labels, T, extents, [mv], level, obstacles)
            overlap[i], landed[i] = over[0], land[0]
            continue
        S = moved_object(occ, labels, T, extents, mv, level).reshape(-1)
        landed[i] = int(S.sum())
        overlap[i] = np.bincount(lab[S & blocking & ~vacated(occ, labels, T, extents, mv, level).reshape(-1)], minlength=N_LABELS)
    return overlap, landed


def placement_in_scene(src_occ, src_labels, scene_occ, scene_labels, T, extents, move, level, axis, sign, lift, obstacles=None):
    """The placement of a group: the group as move (trans = the base) leaves it in the source grid, lowered onto the solid
    obstacle points of the scene that the group does not vacate (a copy vacates nothing) -> placement_turn_oracle.lower's map."""
    S = moved_object(src_occ, src_labels, T, extents, move, level)
    is_obst = np.ones(N_LABELS, dtype=bool) if obstacles is None else np.isin(np.arange(N_LABELS), list(obstacles))
    lab = scene_labels.astype(np.int64)
    O = (scene_occ > np.float32(level)) & is_obst[np.clip(lab, 0, N_LABELS - 1)] & \
        ~vacated(scene_occ, scene_labels, T, extents, move, level)
    return TO.lower(S, O, scene_labels, axis, sign, lift)


def render_apply_moves(raw, rays_o, rays_d, z, moves, T, extents, dim, evaluate, level, voxel, record=None):
    """render_moves_oracle.apply_moves with groups and copies -> (edited copy, evaluated).  record (a list, or None): receives
    each move's decisions (take [n], vacate [n], bool numpy)."""
    out = raw.clone()
    n, s, c = out.shape
    flat = out.reshape(n * s, c)
    pts = RM.RO.sample_points(RM._np(rays_o), RM._np(rays_d), RM._np(z)).reshape(-1, 3)
    dirs = np.repeat(RM._np(rays_d), s, axis=0)
    inv, b = E.grid_index_map(T, extents, dim)
    lev = np.float32(level)
    ev = 0
    for mv in moves:
        if "group" not in mv:
            o2, e2 = CP.render_apply_moves(flat.reshape(n, s, c), rays_o, rays_d, z, [mv], T, extents, dim, evaluate, level, voxel,
                                           record)
            flat.copy_(o2.reshape(n * s, c))
            ev += e2
            continue
        G = group_of(mv)
        trans = np.asarray(mv["trans"], dtype=np.float64)[:3]
        t = E.targets(trans, pts)
        inb = E.in_box(E.index_of(inv, b, t), mv["box"])
        pin = E.in_box(E.index_of(inv, b, pts), mv["box"])
        dev = flat.device
        o_p = RM.occupancy(flat[:, 3], voxel).cpu().numpy()
        l_p = RM.object_labels(flat).cpu().numpy()
        idx = np.nonzero(inb)[0]
        take = np.zeros(flat.shape[0], dtype=bool)
        rows = None
        if idx.size:
            rows = evaluate(t[idx], RM.target_dirs(trans, dirs[idx])).to(dev)
            lt = RM.object_labels(rows).cpu().numpy()
            ot = RM.occupancy(rows[:, 3], voxel).cpu().numpy()
            take[idx] = np.isin(lt, G) & ((ot > lev) | (o_p[idx] <= lev)) & keeps(mv, t[idx], lt)
        vacate = np.zeros(flat.shape[0], dtype=bool)
        if not mv.get("copy"):
            keeps_p = keeps(mv, pts, l_p)
            vacate = ~take & np.isin(l_p, G) & ((keeps_p & pin) | (bool(mv.get("rest_drop", False)) & ~keeps_p))
        if idx.size:
            took = take[idx]
            flat[torch.as_tensor(idx[took], device=dev)] = rows[torch.as_tensor(took, device=dev)]
        flat[torch.as_tensor(np.nonzero(vacate)[0], device=dev), 3] = 0.0
        if record is not None:
            record.append((take, vacate))
        ev += int(idx.size)
    return out, ev


def render_on_depths(rays_o, rays_d, p_coarse, p_fine, z_coarse, z_fine, moves, T, extents, dim, level, voxel, record=None):
    """copy_oracle.render_on_depths with groups: both passes teacher-forced on given depths in the dtype of the state dicts, the
    moves applied by render_apply_moves."""
    dtype = next(iter(p_coarse.values())).dtype
    o, d = rays_o.float(), rays_d.float()
    vd = (d.double() / torch.norm(d.double(), dim=-1, keepdim=True)).to(dtype)
    out = {}
    for tag, p, z in (("coarse", p_coarse, z_coarse), ("fine", p_fine, z_fine)):
        z = z.float()
        pts = o[:, None, :] + d[:, None, :] * z[..., None]
        x = torch.cat([RM.embed(pts.reshape(-1, 3).to(dtype), 10), RM.embed(vd[:, None].expand(pts.shape).reshape(-1, 3), 4)], -1)
        raw = RM.mlp_forward(p, x).reshape(z.shape[0], z.shape[1], -1)
        rec = None if record is None else record.setdefault(tag, [])
        raw, ev = render_apply_moves(raw, o, d, z, moves, T, extents, dim, RM.network_evaluate(p, dtype), level, voxel, rec)
        rgb, w, depth, ins, acc = RM.composite(raw, z.to(dtype), d.to(dtype))
        out.update({"rgb_" + tag: rgb, "weights_" + tag: w, "depth_" + tag: depth, "ins_" + tag: ins, "acc_" + tag: acc,
                    "raw_" + tag: raw, "evaluated_" + tag: ev})
    return out


def object_contacts(occ, labels, level):
    """collide_oracle.object_contacts (faces [3, 128, 128])."""
    return CO.object_contacts(occ, labels, level)
