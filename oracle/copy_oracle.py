"""CPU oracle of copying objects -- TEST INFRASTRUCTURE ONLY (the product package never imports it).

Restates DESIGN.md, "Copying objects" in numpy on top of the edit-sweep, arrangement, collision, placement and moved-render
oracles.  A copy is a move dict with "copy": True.  It takes exactly as the move with the same fields (target, box, piece test,
air clause) and writes the source's label; it never vacates.  So:
  edit / grid edit   edit_sweep_oracle's take with the vacate removed (arrange_oracle's nearest_evaluate for the grid edit); a
                     copy's overwritten[l] counts every solid state point it lands on, its own label's included;
  move_overlap       collide_oracle's counts with nothing vacated: the source's own solid points are obstacles;
  placement          placement_turn_oracle.lower of the moved object onto every solid obstacle point of the scene;
  arrangement        arrange_oracle's greedy order, a copy item placed and applied as a copy;
  moved render       render_moves_oracle's take with the vacate removed."""
import numpy as np
import torch

from oracle import arrange_oracle as A
from oracle import collide_oracle as CO
from oracle import edit_sweep_oracle as E
from oracle import placement_oracle as PO
from oracle import placement_turn_oracle as TO
from oracle import render_moves_oracle as RM

N_LABELS = A.N_LABELS


def take_mask(o, pts, inv, b, move, evaluate, level):
    """The take decisions of one move on flat state occupancies o [n] at points pts [n, 3] -> (take [n] bool, occ_t [n] float32,
    evaluated): edit_sweep_oracle.apply_move's take, unchanged."""
    mv, piece = int(move["label"]), move.get("piece")
    lev = np.float32(level)
    t = E.targets(np.asarray(move["trans"], dtype=np.float64)[:3], pts)
    idx = np.nonzero(E.in_box(E.index_of(inv, b, t), move["box"]))[0]
    take = np.zeros(o.shape[0], dtype=bool)
    occ_t = np.zeros(o.shape[0], dtype=np.float32)
    if idx.size:
        o_t, l_t = evaluate(t[idx])
        occ_t[idx] = o_t
        ok = (np.asarray(l_t) == mv) & ((np.asarray(o_t) > lev) | (o[idx] <= lev))
        if piece is not None:
            ok &= piece.keeps(t[idx])
        take[idx] = ok
    return take, occ_t, int(idx.size)


def apply(o, lab, pts, inv, b, move, evaluate, level):
    """One move or copy on flat grids (edited in place) -> targets evaluated."""
    if not move.get("copy"):
        return E.apply_move(o, lab, pts, inv, b, move, evaluate, level)
    take, occ_t, n = take_mask(o, pts, inv, b, move, evaluate, level)
    o[take] = occ_t[take]
    lab[take] = int(move["label"])
    return n


def edit(occ, labels, T, extents, moves, evaluate, level):
    """edit_sweep_oracle.edit with copies -> (occ, labels, evaluated)."""
    dim = occ.shape[0]
    o, lab = occ.reshape(-1).astype(np.float32).copy(), labels.reshape(-1).astype(np.int64).copy()
    pts = E.sweep_points(T, extents, dim)
    inv, b = E.grid_index_map(T, extents, dim)
    n = sum(apply(o, lab, pts, inv, b, mv, evaluate, level) for mv in moves)
    return o.reshape(occ.shape), lab.reshape(occ.shape).astype(labels.dtype), n


def grid_edit(src_occ, src_labels, occ, labels, T, extents, moves, level):
    """arrange_oracle.grid_edit with copies -> (occ, labels, landed int64 [n], overwritten int64 [n, 128])."""
    landed = np.zeros(len(moves), dtype=np.int64)
    overwritten = np.zeros((len(moves), N_LABELS), dtype=np.int64)
    state_o, state_l = occ.copy(), labels.copy()
    dim = occ.shape[0]
    pts = E.sweep_points(T, extents, dim)
    inv, b = E.grid_index_map(T, extents, dim)
    ev = A.nearest_evaluate(src_occ.astype(np.float32), src_labels.astype(np.int64), inv, b)
    lev = np.float32(level)
    for i, mv in enumerate(moves):
        if not mv.get("copy"):
            state_o, state_l, land, over = A.grid_edit(src_occ, src_labels, state_o, state_l, T, extents, [mv], level)
            landed[i], overwritten[i] = land[0], over[0]
            continue
        o, lab = state_o.reshape(-1).astype(np.float32).copy(), state_l.reshape(-1).astype(np.int64).copy()
        take, occ_t, _ = take_mask(o, pts, inv, b, mv, ev, level)
        solid_take = take & (occ_t > lev)
        landed[i] = int(solid_take.sum())
        overwritten[i] = np.bincount(lab[solid_take & (o > lev)], minlength=N_LABELS)
        apply(o, lab, pts, inv, b, mv, ev, level)
        state_o, state_l = o.reshape(occ.shape), lab.reshape(occ.shape).astype(labels.dtype)
    return state_o, state_l, landed, overwritten


def move_overlap(occ, labels, T, extents, moves, level, obstacles=None):
    """collide_oracle.move_overlap with copies (each candidate on its own) -> (overlap int64 [n, 128], landed int64 [n])."""
    overlap = np.zeros((len(moves), N_LABELS), dtype=np.int64)
    landed = np.zeros(len(moves), dtype=np.int64)
    dim = occ.shape[0]
    o, lab = occ.reshape(-1).astype(np.float32), labels.reshape(-1).astype(np.int64)
    pts = E.sweep_points(T, extents, dim)
    inv, b = E.grid_index_map(T, extents, dim)
    is_obst = np.ones(N_LABELS, dtype=bool) if obstacles is None else np.isin(np.arange(N_LABELS), list(obstacles))
    blocking = (o > np.float32(level)) & is_obst[np.clip(lab, 0, N_LABELS - 1)]
    for i, mv in enumerate(moves):
        if not mv.get("copy"):
            over, land = CO.move_overlap(occ, labels, T, extents, [mv], level, obstacles)
            overlap[i], landed[i] = over[0], land[0]
            continue
        S = TO.moved_object(occ, labels, T, extents, mv["label"], level, mv["trans"], mv["box"], mv.get("piece")).reshape(-1)
        landed[i] = int(S.sum())
        overlap[i] = np.bincount(lab[S & blocking], minlength=N_LABELS)
    return overlap, landed


def placement_in_scene(src_occ, src_labels, scene_occ, scene_labels, T, extents, label, level, axis, sign, lift, base, box,
                       piece=None, obstacles=None):
    """The placement of a copy: the object as `base` leaves it in the source grid, lowered onto every solid obstacle point of
    the scene (nothing vacated: sets() of a label no point carries)."""
    S = TO.moved_object(src_occ, src_labels, T, extents, label, level, base, box, piece)
    _, O = PO.sets(scene_occ, scene_labels, T, extents, -1, level, None, False, obstacles)
    return TO.lower(S, O, scene_labels, axis, sign, lift)


def arrange(occ, labels, T, extents, items, down, level, max_tests=64):
    """arrange_oracle.arrange with copy items (key "copy") -> (occ, labels, [per item None or dict(turn, offset, drop, trans)])."""
    from fractions import Fraction
    dim = occ.shape[0]
    axis, sign = PO.down_axis(T, extents, down)
    Am, _ = A.grid_affine(T, dim, extents)
    h = [a for a in range(3) if a != axis]
    state_o, state_l = occ.copy(), labels.copy()
    pts = E.sweep_points(T, extents, dim)
    chosen = []
    for it in items:
        label, piece, lift, copy = int(it["label"]), it.get("piece"), int(it.get("lift", 0)), bool(it.get("copy", False))
        keep = None if piece is None else piece.keeps(pts).reshape(occ.shape)
        S0, _ = PO.sets(occ, labels, T, extents, label, level, piece)
        src_box = E.solid_box(occ, labels, label, level, 2, keep)
        idx = np.argwhere(S0)
        turns = it.get("turns")
        if turns is None:
            bases = [np.eye(4)]
        else:
            box = [int(x) for a in range(3) for x in (idx[:, a].min(), idx[:, a].max())]
            centre = [Fraction(int(s), idx.shape[0]) for s in idx.sum(0)]
            bases = [TO.turn_base(T, extents, dim, axis, centre, box, 360.0 * k / turns) for k in range(turns)]
        maps = []
        for k, base in enumerate(bases):
            if base is None:
                continue
            S = TO.moved_object(occ, labels, T, extents, label, level, base, src_box, piece)
            if not S.any() or np.argwhere(PO.to_columns(S, axis, sign))[:, 2].max() + lift > dim - 1:
                continue
            if copy:
                m = placement_in_scene(occ, labels, state_o, state_l, T, extents, label, level, axis, sign, lift, base, src_box,
                                       piece, it.get("obstacles"))
            else:
                m = A.placement_in_scene(occ, labels, state_o, state_l, T, extents, label, level, axis, sign, lift, base, src_box,
                                         piece, it.get("rest_drop", False), it.get("obstacles"))
            maps.append((k, m))
        rows = A.candidates(maps, it["near"], it.get("on"), T, extents, axis, sign, dim)
        pick = None
        for r in rows[:max_tests]:
            k, u, v = int(r[1]), int(r[2]), int(r[3])
            m = dict(maps)[k]
            if PO.stable(m, u, v) or not it.get("stable", True):
                pick = (k, u, v, m)
                break
        if pick is None:
            chosen.append(None)
            continue
        k, u, v, m = pick
        drop = int(m["drop"][u - m["offset_lo"][0], v - m["offset_lo"][1]])
        delta = np.zeros(3)
        delta[h[0]], delta[h[1]] = u, v
        delta[axis] = -sign * (lift - drop)
        trans = bases[k] @ A._translate(-(Am @ delta)) if turns is not None else A._translate(-(Am @ delta))
        move = {"label": label, "trans": trans, "box": src_box, "piece": piece, "rest_drop": it.get("rest_drop", False),
                "copy": copy}
        state_o, state_l, _, _ = grid_edit(occ, labels, state_o, state_l, T, extents, [move], level)
        chosen.append({"turn": None if turns is None else 360.0 * k / turns, "offset": (u, v), "drop": drop, "trans": trans})
    return state_o, state_l, chosen


def render_apply_moves(raw, rays_o, rays_d, z, moves, T, extents, dim, evaluate, level, voxel, record=None):
    """render_moves_oracle.apply_moves with copies: a copy's take as the move's, and no vacate -> (edited copy, evaluated).
    record (a list, or None): receives each move's decisions (take [n], vacate [n], bool numpy; a copy's vacate all False)."""
    out = raw.clone()
    n, s, c = out.shape
    flat = out.reshape(n * s, c)
    pts = RM.RO.sample_points(RM._np(rays_o), RM._np(rays_d), RM._np(z)).reshape(-1, 3)
    dirs = np.repeat(RM._np(rays_d), s, axis=0)
    inv, b = E.grid_index_map(T, extents, dim)
    ev = 0
    for mv in moves:
        if not mv.get("copy"):
            ev += RM.apply_move(flat, pts, dirs, mv, inv, b, evaluate, level, voxel, record)
            continue
        rec = []
        before = flat.clone()
        ev += RM.apply_move(flat, pts, dirs, mv, inv, b, evaluate, level, voxel, rec)
        take, vacate = rec[0]
        undo = torch.as_tensor(np.nonzero(vacate & ~take)[0], device=flat.device)
        flat[undo] = before[undo]                                  # the move's vacate, undone: a copy vacates nothing
        if record is not None:
            record.append((take, np.zeros_like(vacate)))
    return out, ev


def render_on_depths(rays_o, rays_d, p_coarse, p_fine, z_coarse, z_fine, moves, T, extents, dim, level, voxel, record=None):
    """render_moves_oracle.render_on_depths with copies: both passes teacher-forced on given depths, the network p (state dicts,
    their dtype) on the fp32 sample points and the unit view directions, the moves and copies applied by render_apply_moves
    (targets through render_moves_oracle.network_evaluate), then dmnerf_oracle's composite in that dtype.  record: {"coarse":
    [...], "fine": [...]} of the decisions, or None."""
    dtype = next(iter(p_coarse.values())).dtype
    o, d = rays_o.float(), rays_d.float()
    vd = (d.double() / torch.norm(d.double(), dim=-1, keepdim=True)).to(dtype)
    out = {}
    for tag, p, z in (("coarse", p_coarse, z_coarse), ("fine", p_fine, z_fine)):
        z = z.float()
        pts = o[:, None, :] + d[:, None, :] * z[..., None]                     # the prologue's fp32 point
        x = torch.cat([RM.embed(pts.reshape(-1, 3).to(dtype), 10), RM.embed(vd[:, None].expand(pts.shape).reshape(-1, 3), 4)], -1)
        raw = RM.mlp_forward(p, x).reshape(z.shape[0], z.shape[1], -1)
        rec = None if record is None else record.setdefault(tag, [])
        raw, ev = render_apply_moves(raw, o, d, z, moves, T, extents, dim, RM.network_evaluate(p, dtype), level, voxel, rec)
        rgb, w, depth, ins, acc = RM.composite(raw, z.to(dtype), d.to(dtype))
        out.update({"rgb_" + tag: rgb, "weights_" + tag: w, "depth_" + tag: depth, "ins_" + tag: ins, "acc_" + tag: acc,
                    "raw_" + tag: raw, "evaluated_" + tag: ev})
    return out
