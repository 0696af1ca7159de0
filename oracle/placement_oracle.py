"""CPU oracle of object placement -- TEST INFRASTRUCTURE ONLY (the product package never imports it).

Restates DESIGN.md, "Object placement" by brute force in numpy, on edit_sweep_oracle's sweep points and pieces and
collide_oracle's vacate rule:
  object S     labels == label, occ > level, kept by the piece at the fp32 sweep point (every point without one);
  obstacles O  occ > level, label among the obstacles, not vacated (label == mv and in the piece, or rest dropped);
  heights      y = idx_axis (sign -1) or dim - 1 - idx_axis (sign +1: +e_axis points down);
  drop         per offset (u, v): S + (u, v, lift) overlaps O -> -1; else lowered one voxel at a time while the next step
               neither overlaps O nor reaches below height 0;
  support      at rest, the object points with an obstacle point directly below: their count, and the label below most of
               them (ties: the lowest label; -1 without any).
It lowers the whole voxel set step by step and never uses the run argument of the kernels.  Stability: the centre of mass (an
exact rational) against the closed convex hull of the support cells, with Fractions."""
from fractions import Fraction
from functools import cmp_to_key

import numpy as np

from oracle import edit_sweep_oracle as E

N_LABELS = 128


def down_axis(T, extents, down):
    """(axis, sign) of the index axis closest to +-down (network frame): sign +1 when +e_axis points down."""
    inv, _ = E.grid_index_map(T, extents, 2)
    A = np.linalg.inv(inv)
    dirs = (A / np.linalg.norm(A, axis=0)).T
    d = np.asarray(down, dtype=np.float64)
    dots = dirs @ (d / np.linalg.norm(d))
    a = int(np.argmax(np.abs(dots)))
    return a, (1 if dots[a] > 0 else -1)


def to_columns(grid, axis, sign):
    """A [dim]^3 grid (C order of (i, j, k)) as [h1, h2, y]."""
    h = [a for a in range(3) if a != axis]
    g = np.transpose(grid, (h[0], h[1], axis))
    return g[:, :, ::-1] if sign > 0 else g


def sets(occ, labels, T, extents, label, level, piece=None, rest_drop=False, obstacles=None):
    """(S, O) bool [dim]^3 in grid order."""
    dim = occ.shape[0]
    o, lab = occ.reshape(-1).astype(np.float32), labels.reshape(-1).astype(np.int64)
    solid = o > np.float32(level)
    keep = np.ones(o.shape[0], dtype=bool) if piece is None else piece.keeps(E.sweep_points(T, extents, dim))
    S = solid & (lab == label) & keep
    is_obst = np.ones(N_LABELS, dtype=bool) if obstacles is None else np.isin(np.arange(N_LABELS), list(obstacles))
    vacated = (lab == label) & (keep | bool(rest_drop))
    O = solid & is_obst[np.clip(lab, 0, N_LABELS - 1)] & ~vacated
    return S.reshape(occ.shape), O.reshape(occ.shape)


def placement_map(occ, labels, T, extents, label, level, axis, sign, lift, piece=None, rest_drop=False, obstacles=None):
    """Brute force -> dict(drop, contacts, support [U, V], offset_lo, points [n, 3] (h1, h2, y), O, L ([h1, h2, y] grids),
    centre (Fractions, (h1, h2, y)))."""
    dim = occ.shape[0]
    S, O = sets(occ, labels, T, extents, label, level, piece, rest_drop, obstacles)
    Sc, Oc, Lc = to_columns(S, axis, sign), to_columns(O, axis, sign), to_columns(labels.astype(np.int64), axis, sign)
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
                counts = np.bincount(Lc[rest[:, 0], rest[:, 1], rest[:, 2]], minlength=N_LABELS)
                support[iu, iv] = int(np.argmax(counts))              # first maximum: the lowest label
    n = pts.shape[0]
    return {"drop": drop, "contacts": contacts, "support": support, "offset_lo": (-int(lo[0]), -int(lo[1])), "points": pts,
            "O": Oc, "L": Lc, "centre": [Fraction(int(s), n) for s in pts.sum(0)], "lift": lift}


def support_cells(m, u, v):
    """The support cells at offset (u, v): [(h1, h2, label below)] of the resting points with an obstacle below, in (column,
    height) order."""
    iu, iv = u - m["offset_lo"][0], v - m["offset_lo"][1]
    d = int(m["drop"][iu, iv])
    assert d >= 0
    p = m["points"] + np.array([u, v, m["lift"] - d])
    p = p[p[:, 2] >= 1]
    O = m["O"]
    rest = p[O[p[:, 0], p[:, 1], p[:, 2] - 1]]
    rest = rest[np.lexsort((rest[:, 2], rest[:, 1], rest[:, 0]))]
    return [(int(a), int(b), int(m["L"][a, b, c - 1])) for a, b, c in rest]


def in_hull(cells, point):
    """Whether `point` (2 Fractions) lies in the closed convex hull of the integer cells [(a, b), ...], exactly: it does unless
    the vectors from it to the cells leave an angular gap wider than a half turn (then a line through it separates them).  The
    vectors are scaled to integers and sorted by angle with integer cross products."""
    x, y = Fraction(point[0]), Fraction(point[1])
    den = x.denominator * y.denominator
    X, Y = int(x * den), int(y * den)
    vs = [(int(a) * den - X, int(b) * den - Y) for a, b in set((int(a), int(b)) for a, b in cells)]
    if not vs:
        return False
    if any(v == (0, 0) for v in vs):
        return True

    def cross(a, b):
        return a[0] * b[1] - a[1] * b[0]

    def half(v):
        return 0 if v[1] > 0 or (v[1] == 0 and v[0] > 0) else 1
    vs.sort(key=cmp_to_key(lambda a, b: (half(a) - half(b)) or (-1 if cross(a, b) > 0 else (1 if cross(a, b) < 0 else 0))))
    if all(cross(vs[0], v) == 0 and vs[0][0] * v[0] + vs[0][1] * v[1] > 0 for v in vs):
        return False                                   # one direction: a full turn of gap
    return all(cross(vs[i], vs[(i + 1) % len(vs)]) >= 0 for i in range(len(vs)))


def stable(m, u, v):
    """The placement at (u, v) is stable: the centre of mass's horizontal projection in the closed hull of its support cells."""
    cells = [(a, b) for a, b, _ in support_cells(m, u, v)]
    return in_hull(cells, (m["centre"][0] + u, m["centre"][1] + v))


def delta(axis, sign, lift, u, v, drop):
    """The index displacement of the placement: (u, v) on the horizontal axes, lift - drop in height."""
    h = [a for a in range(3) if a != axis]
    d = np.zeros(3, dtype=np.int64)
    d[h[0]], d[h[1]] = u, v
    d[axis] = -sign * (lift - drop)
    return d
