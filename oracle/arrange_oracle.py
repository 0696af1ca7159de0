"""CPU oracle of arranging objects -- TEST INFRASTRUCTURE ONLY (the product package never imports it).

Restates DESIGN.md, "Arranging objects" in numpy on top of the edit-sweep, collision and placement oracles:
  grid edit    edit_sweep_oracle's take / vacate with the network replaced by the unedited (source) grid at rint(u) of every
               target (nearest_evaluate), applied to a state grid; per move, by brute force over the grid points, landed = the
               takes whose target is solid and overwritten[l] = those of them on a solid state point of label l that the move does
               not vacate (label mv and in the piece -- every point without one -- or rest dropped);
  in a scene   the object S_base from the source grid (placement_turn_oracle.moved_object), the obstacles O and the labels under
               it from the scene (placement_oracle.sets), lowered by placement_turn_oracle.lower;
  arrangement  the items in order: the candidates of every turn in place_object's order (distance of the placed centre from
               `near` across down, then turn, then (u, v)), the first stable one (placement_oracle.stable) among the nearest
               max_tests -- or the first with stable False -- applied to the state by the grid edit with the default box."""
from fractions import Fraction

import numpy as np

from oracle import edit_sweep_oracle as E
from oracle import placement_oracle as PO
from oracle import placement_turn_oracle as TO

N_LABELS = 128


def nearest_evaluate(occ, labels, inv, b):
    """evaluate() for any target in the grid: the unedited grid at rint(u)."""
    def f(t):
        i = np.rint(E.index_of(inv, b, t)).astype(np.int64)
        return occ[i[:, 0], i[:, 1], i[:, 2]], labels[i[:, 0], i[:, 1], i[:, 2]]
    return f


def grid_edit(src_occ, src_labels, occ, labels, T, extents, moves, level):
    """The moves (edit_sweep_oracle's dicts: label, trans, box, piece, rest_drop) applied in order to copies of the state occ /
    labels, every target read from src_occ / src_labels -> (occ, labels, landed int64 [n], overwritten int64 [n, 128])."""
    dim = occ.shape[0]
    o, lab = occ.reshape(-1).astype(np.float32).copy(), labels.reshape(-1).astype(np.int64).copy()
    pts = E.sweep_points(T, extents, dim)
    inv, b = E.grid_index_map(T, extents, dim)
    ev = nearest_evaluate(src_occ.astype(np.float32), src_labels.astype(np.int64), inv, b)
    lev = np.float32(level)
    landed = np.zeros(len(moves), dtype=np.int64)
    overwritten = np.zeros((len(moves), N_LABELS), dtype=np.int64)
    for i, mv in enumerate(moves):
        label, piece = int(mv["label"]), mv.get("piece")
        t = E.targets(np.asarray(mv["trans"], dtype=np.float64)[:3], pts)
        inb = E.in_box(E.index_of(inv, b, t), mv["box"])
        take = np.zeros(o.shape[0], dtype=bool)
        o_t = np.zeros(o.shape[0], dtype=np.float32)
        for p in np.nonzero(inb)[0]:                               # point by point: the count's own restatement
            ot, lt = ev(t[p:p + 1])
            o_t[p] = ot[0]
            ok = int(lt[0]) == label and (ot[0] > lev or o[p] <= lev)
            take[p] = ok and (piece is None or bool(piece.keeps(t[p:p + 1])[0]))
        in_piece = np.ones(o.shape[0], dtype=bool) if piece is None else piece.keeps(pts)
        vacated = (lab == label) & (in_piece | bool(mv.get("rest_drop", False)))
        solid_take = take & (o_t > lev)
        landed[i] = int(solid_take.sum())
        hit = solid_take & (o > lev) & ~vacated
        overwritten[i] = np.bincount(lab[hit], minlength=N_LABELS)
        E.apply_move(o, lab, pts, inv, b, mv, ev, level)
    return o.reshape(occ.shape), lab.reshape(occ.shape).astype(labels.dtype), landed, overwritten


def placement_in_scene(src_occ, src_labels, scene_occ, scene_labels, T, extents, label, level, axis, sign, lift, base, box,
                       piece=None, rest_drop=False, obstacles=None):
    """placement_turn_oracle.lower of the object as `base` leaves it in the source grid, onto the scene's obstacles."""
    S = TO.moved_object(src_occ, src_labels, T, extents, label, level, base, box, piece)
    _, O = PO.sets(scene_occ, scene_labels, T, extents, label, level, piece, rest_drop, obstacles)
    return TO.lower(S, O, scene_labels, axis, sign, lift)


def grid_affine(T, dim, extents):
    """objects.grid_affine restated: p = A idx + b."""
    T = np.asarray(T, dtype=np.float64)
    ext = np.asarray(extents, dtype=np.float64)
    R, t = T[:3, :3], T[:3, 3]
    return E.S @ (R * (ext / (dim - 1))[None, :]), E.S @ (t - R @ (ext / 2.0))


def _translate(v):
    m = np.eye(4)
    m[:3, 3] = v
    return m


def _grid_centre(m, axis, sign, dim):
    """A lowered map's centre (h1, h2, y) as grid-order index Fractions."""
    h = [a for a in range(3) if a != axis]
    c = [None] * 3
    c[h[0]], c[h[1]] = m["centre"][0], m["centre"][1]
    c[axis] = dim - 1 - m["centre"][2] if sign > 0 else m["centre"][2]
    return c


def candidates(maps, near, on, T, extents, axis, sign, dim):
    """place_object's candidate order over maps [(turn index, map)] -> rows (distance, turn, u, v)."""
    A, b = grid_affine(T, dim, extents)
    n = A[:, axis] / np.linalg.norm(A[:, axis])
    h = [a for a in range(3) if a != axis]
    rows = [np.zeros((0, 4))]
    for t, m in maps:
        ok = (m["drop"] >= 0) & (m["support"] >= 0)
        if on is not None:
            ok &= np.isin(m["support"], sorted(on))
        iu, iv = np.nonzero(ok)
        u, v = iu + m["offset_lo"][0], iv + m["offset_lo"][1]
        cm = np.array([float(x) for x in _grid_centre(m, axis, sign, dim)])
        delta = np.zeros((iu.size, 3))
        delta[:, h[0]], delta[:, h[1]] = u, v
        delta[:, axis] = -sign * (m["lift"] - m["drop"][iu, iv])
        gap = (cm[None, :] + delta) @ A.T + b - np.asarray(near, dtype=np.float64)[None, :]
        gap -= np.outer(gap @ n, n)
        rows.append(np.stack([np.linalg.norm(gap, axis=1), np.full(iu.size, t), u, v], 1))
    rows = np.concatenate(rows)
    return rows[np.lexsort((rows[:, 3], rows[:, 2], rows[:, 1], rows[:, 0]))]


def arrange(occ, labels, T, extents, items, down, level, max_tests=64):
    """The arrangement of `items` (dicts: label, near, and optionally on, turns (an integer K), stable, lift, piece (E.Piece),
    rest_drop, obstacles) -> (occ, labels, [per item None or dict(turn, offset, drop, trans)])."""
    dim = occ.shape[0]
    axis, sign = PO.down_axis(T, extents, down)
    A, _ = grid_affine(T, dim, extents)
    h = [a for a in range(3) if a != axis]
    state_o, state_l = occ.copy(), labels.copy()
    pts = E.sweep_points(T, extents, dim)
    chosen = []
    for it in items:
        label, piece, lift = int(it["label"]), it.get("piece"), int(it.get("lift", 0))
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
            maps.append((k, placement_in_scene(occ, labels, state_o, state_l, T, extents, label, level, axis, sign, lift, base,
                                               src_box, piece, it.get("rest_drop", False), it.get("obstacles"))))
        rows = candidates(maps, it["near"], it.get("on"), T, extents, axis, sign, dim)
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
        trans = bases[k] @ _translate(-(A @ delta)) if turns is not None else _translate(-(A @ delta))
        move = {"label": label, "trans": trans, "box": src_box, "piece": piece, "rest_drop": it.get("rest_drop", False)}
        state_o, state_l, _, _ = grid_edit(occ, labels, state_o, state_l, T, extents, [move], level)
        chosen.append({"turn": None if turns is None else 360.0 * k / turns, "offset": (u, v), "drop": drop, "trans": trans})
    return state_o, state_l, chosen
