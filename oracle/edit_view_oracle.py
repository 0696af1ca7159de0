"""CPU oracle of colouring an edited view -- TEST INFRASTRUCTURE ONLY (the product package never imports it).

Restates DESIGN.md, "Colouring an edited view" in numpy on top of deform_oracle (targets, take_mask, the pull and its
direction), group_oracle's vacate, region pieces (edit_sweep_oracle.Piece) and grid_cast_oracle's walk.  Moves are the dicts of
deform_oracle (label, trans, box, and optionally piece, applies, rest_drop, copy, group, deform), applied in order:
  provenance   per hit voxel q: (o, l) = source[q]; for each move k at q's sweep point p, deform_oracle.take_mask (the target
               read from the source at its nearest index) and group_oracle.vacate_mask; a take sets (o, l) and m* = k, a vacate
               sets o = 0.  m* = -1 where no move took;
  consistency  the replay's (o, l) against the viewed grid's (occ[q], labels[q]), the occupancy by its bits;
  colour       x = o + depth d (fp32, multiply then add); for m* >= 0 the point is the target of x under move m*
               (deform_oracle.targets) and the direction trans[:3, :3] d in fp64, pulled back by deform_oracle.direction at x's
               pulled point for a deformed move, rounded once to fp32 and not normalised; for m* = -1, x and d."""
import numpy as np

from oracle import deform_oracle as DO
from oracle import edit_sweep_oracle as E
from oracle import grid_cast_oracle as G
from oracle import group_oracle as GO


def provenance(src_occ, src_labels, T, extents, moves, voxel, level):
    """The moves replayed at the hit voxels voxel [n] (C-order index, -1: no hit) -> (move int32 [n], occ float32 [n], label int64
    [n]); rays without a hit get -1, 0 and -1."""
    dim = src_occ.shape[0]
    voxel = np.asarray(voxel, dtype=np.int64).reshape(-1)
    hit = np.nonzero(voxel >= 0)[0]
    q = voxel[hit]
    src_o, src_l = np.asarray(src_occ, dtype=np.float32).reshape(-1), np.asarray(src_labels).reshape(-1).astype(np.int64)
    pts = E.sweep_points(T, extents, dim)[q]
    inv, b = E.grid_index_map(T, extents, dim)
    ev = DO.nearest_evaluate(src_o.reshape(src_occ.shape), src_l.reshape(src_occ.shape), inv, b)
    o, lab = src_o[q].copy(), src_l[q].copy()
    m = np.full(q.shape[0], -1, dtype=np.int32)
    for k, mv in enumerate(moves):
        take, occ_t, lab_t, _ = DO.take_mask(o, pts, inv, b, mv, ev, level)
        vacate = GO.vacate_mask(o, lab, pts, mv, level, take)
        o[take], lab[take] = occ_t[take], lab_t[take]
        o[vacate] = 0.0
        m[take] = k
    move = np.full(voxel.shape[0], -1, dtype=np.int32)
    occ_r = np.zeros(voxel.shape[0], dtype=np.float32)
    lab_r = np.full(voxel.shape[0], -1, dtype=np.int64)
    move[hit], occ_r[hit], lab_r[hit] = m, o, lab
    return move, occ_r, lab_r


def mismatched(occ, labels, voxel, occ_r, lab_r):
    """The hits whose replay (occ_r, lab_r) differs from the viewed grid at the hit voxel, the occupancy by its bits -> bool [n]."""
    voxel = np.asarray(voxel, dtype=np.int64).reshape(-1)
    hit = voxel >= 0
    q = np.where(hit, voxel, 0)
    o = np.asarray(occ, dtype=np.float32).reshape(-1)[q]
    lab = np.asarray(labels).reshape(-1).astype(np.int64)[q]
    return hit & ((o.view(np.int32) != occ_r.view(np.int32)) | (lab != lab_r))


def colour_rays(rays_o, rays_d, depth, voxel, move, moves):
    """The colour point [n, 3] float32 (NaN without a hit) and the direction [n, 3] float32, not normalised (0 without a hit), of
    the rays with cast depth [n], hit voxel [n] and provenance move [n]."""
    o = np.asarray(rays_o, dtype=np.float32).reshape(-1, 3)
    d = np.asarray(rays_d, dtype=np.float32).reshape(-1, 3)
    depth = np.asarray(depth, dtype=np.float32).reshape(-1)
    hit = np.asarray(voxel).reshape(-1) >= 0
    with np.errstate(all="ignore"):
        x = (o + (depth[:, None] * d).astype(np.float32)).astype(np.float32)
    point = np.where(hit[:, None], x, np.float32(np.nan)).astype(np.float32)
    dirs = np.where(hit[:, None], d, np.float32(0.0)).astype(np.float32)
    for k, mv in enumerate(moves):
        rows = np.nonzero(hit & (np.asarray(move).reshape(-1) == k))[0]
        if not rows.size:
            continue
        trans = np.asarray(mv["trans"], dtype=np.float64)[:3]
        point[rows] = DO.targets(mv, x[rows])
        dd = d[rows].astype(np.float64)
        w = np.stack([(trans[a, 0] * dd[:, 0] + trans[a, 1] * dd[:, 1]) + trans[a, 2] * dd[:, 2] for a in range(3)], -1)
        if mv.get("deform") is not None:
            _, st = DO.pull(mv["deform"], DO.moved(trans, x[rows]))
            w = DO.direction(mv["deform"], st, w)
        dirs[rows] = w.astype(np.float32)
    return point, dirs


def edit_view(occ, labels, src_occ, src_labels, T, extents, rays_o, rays_d, near, far, moves, level, cast=None):
    """The whole rule on the viewed grid occ / labels: the cast (grid_cast_oracle.cast, or `cast` given as its dict), the
    provenance, the mismatched hits and the colour point and direction -> dict(cast, move, mismatched, point, dir)."""
    c = cast if cast is not None else G.cast(occ, labels, T, extents, rays_o, rays_d, near, far, level)
    move, occ_r, lab_r = provenance(src_occ, src_labels, T, extents, moves, c["voxel"], level)
    bad = mismatched(occ, labels, c["voxel"], occ_r, lab_r)
    point, dirs = colour_rays(rays_o, rays_d, c["t"], c["voxel"], move, moves)
    return dict(cast=c, move=move, mismatched=bad, point=point, dir=dirs)
