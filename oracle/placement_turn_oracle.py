"""CPU oracle of turned placements -- TEST INFRASTRUCTURE ONLY (the product package never imports it).

Restates DESIGN.md, "Turned placements" in numpy on top of placement_oracle and of the collision checks' target and
nearest-index functions (edit_sweep_oracle):
  object S_base  src(p): q = rint(inv (t - b)) of t = fp32(base p) in the source box B, labels[q] == label, occ[q] > level and
                 (no piece or the piece keeps t); the sweep's grid points only, so points carried outside the grid are lost;
  obstacles O    placement_oracle's, from the object as it lies (the points the move vacates are its own points);
  the map        the same brute-force lowering as placement_oracle, over S_base;
  turn_base      the turn about the down index axis, restated from the rule (Rodrigues' formula, exact at quarter turns);
  tie_distance   per grid point, how close the fp64 index coordinate of its target is to a half-integer: where it is about one
                 fp32 rounding of t or less, a different operation order can pick the other nearest index.
The result of placement_map has placement_oracle's keys, so that its support_cells and stable apply unchanged."""
from fractions import Fraction

import numpy as np

from oracle import edit_sweep_oracle as E
from oracle import placement_oracle as PO

N_LABELS = PO.N_LABELS


def moved_object(occ, labels, T, extents, label, level, base, box, piece=None):
    """S_base, bool [dim]^3 in grid order: the grid points p with src(p) under `base`."""
    dim = occ.shape[0]
    o, lab = occ.reshape(-1).astype(np.float32), labels.reshape(-1).astype(np.int64)
    pts = E.sweep_points(T, extents, dim)
    inv, b = E.grid_index_map(T, extents, dim)
    t = E.targets(np.asarray(base, dtype=np.float64)[:3], pts)
    u = E.index_of(inv, b, t)
    src = E.in_box(u, box)
    q = np.rint(u[src]).astype(np.int64)
    qi = (q[:, 0] * dim + q[:, 1]) * dim + q[:, 2]
    ok = (lab[qi] == int(label)) & (o[qi] > np.float32(level))
    if piece is not None:
        ok &= piece.keeps(t[src])
    src[np.nonzero(src)[0]] = ok
    return src.reshape(occ.shape)


def lower(S, O, labels, axis, sign, lift):
    """placement_oracle's brute-force lowering of the voxel set S (grid order) onto the obstacles O."""
    dim = S.shape[0]
    Sc, Oc, Lc = PO.to_columns(S, axis, sign), PO.to_columns(O, axis, sign), PO.to_columns(labels.astype(np.int64), axis, sign)
    pts = np.argwhere(Sc)
    assert pts.size, "the object has no points"
    lo, hi = pts.min(0), pts.max(0)
    assert hi[2] + lift <= dim - 1
    U, V = dim - (hi[0] - lo[0]), dim - (hi[1] - lo[1])
    drop = np.full((U, V), -1, dtype=np.int64)
    contacts = np.zeros((U, V), dtype=np.int64)
    support = np.full((U, V), -1, dtype=np.int64)
    for iu in range(U):
        for iv in range(V):
            p = pts + np.array([iu - lo[0], iv - lo[1], lift])
            if Oc[p[:, 0], p[:, 1], p[:, 2]].any():
                continue
            h = 0
            while p[:, 2].min() - 1 >= 0 and not Oc[p[:, 0], p[:, 1], p[:, 2] - 1].any():
                p = p - np.array([0, 0, 1])
                h += 1
            drop[iu, iv] = h
            under = p[p[:, 2] >= 1] - np.array([0, 0, 1])
            rest = under[Oc[under[:, 0], under[:, 1], under[:, 2]]]
            contacts[iu, iv] = rest.shape[0]
            if rest.shape[0]:
                support[iu, iv] = int(np.argmax(np.bincount(Lc[rest[:, 0], rest[:, 1], rest[:, 2]], minlength=N_LABELS)))
    n = pts.shape[0]
    return {"drop": drop, "contacts": contacts, "support": support, "offset_lo": (-int(lo[0]), -int(lo[1])), "points": pts,
            "O": Oc, "L": Lc, "centre": [Fraction(int(s), n) for s in pts.sum(0)], "lift": lift}


def placement_map(occ, labels, T, extents, label, level, axis, sign, lift, base=None, box=None, piece=None, rest_drop=False,
                  obstacles=None):
    """placement_oracle.placement_map of the object as `base` leaves it (base None: as it lies, placement_oracle's S)."""
    S, O = PO.sets(occ, labels, T, extents, label, level, piece, rest_drop, obstacles)
    if base is not None:
        S = moved_object(occ, labels, T, extents, label, level, base, box, piece)
    return lower(S, O, labels, axis, sign, lift)


def turn_base(T, extents, dim, axis, centre, box, angle):
    """The base of a turn by `angle` degrees about the down index axis, or None when it does not fit: the pivot is the grid
    point nearest `centre` (index space), moved by whole voxels to the grid's middle column; R turns about A[:, axis] / |.|;
    the object lands at L(x) = R (x - P) + P + A s and the base is L^-1.  The fit: the box grown by half a voxel, its corners
    carried by L, inside [-0.5, dim - 0.5] on the horizontal axes."""
    inv, b = E.grid_index_map(T, extents, dim)
    A = np.linalg.inv(inv)
    n = A[:, axis] / np.linalg.norm(A[:, axis])
    quarter, r = divmod(float(angle), 90.0)
    c, s = ((1.0, 0.0), (0.0, 1.0), (-1.0, 0.0), (0.0, -1.0))[int(quarter) % 4] if r == 0 else \
        (np.cos(np.radians(angle)), np.sin(np.radians(angle)))
    K = np.array([[0.0, -n[2], n[1]], [n[2], 0.0, -n[0]], [-n[1], n[0], 0.0]])
    R = c * np.eye(3) + s * K + (1.0 - c) * np.outer(n, n)
    pivot = np.array([np.floor(Fraction(x) + Fraction(1, 2)) for x in centre], dtype=np.float64)
    shift = np.array([0.0 if a == axis else (dim - 1) // 2 - pivot[a] for a in range(3)])
    P = A @ pivot + b
    h = [a for a in range(3) if a != axis]
    for k in range(8):
        corner = np.array([box[2 * a + 1] + 0.5 if (k >> a) & 1 else box[2 * a] - 0.5 for a in range(3)], dtype=np.float64)
        landed = inv @ (R @ (A @ corner + b - P) + P + A @ shift - b)
        if (landed[h] < -0.5 - 1e-9).any() or (landed[h] > dim - 0.5 + 1e-9).any():
            return None
    base = np.eye(4)
    base[:3, :3] = R.T
    base[:3, 3] = P - R.T @ (P + A @ shift)
    return base


def tie_distance(T, extents, dim, trans):
    """Per grid point (C order), min over the axes of | |u - floor(u)| - 1/2 | for u = inv (fp32(trans p) - b): 0 at an exact
    nearest-index tie."""
    pts = E.sweep_points(T, extents, dim)
    inv, b = E.grid_index_map(T, extents, dim)
    u = E.index_of(inv, b, E.targets(np.asarray(trans, dtype=np.float64)[:3], pts))
    return np.abs((u - np.floor(u)) - 0.5).min(axis=1)


def near_ties(T, extents, dim, trans, tol=1e-5):
    """The grid points whose target lies within `tol` index units of a nearest-index tie (about 40 fp32 roundings of t at
    dim 33 and extents 4)."""
    return int((tie_distance(T, extents, dim, trans) < tol).sum())
