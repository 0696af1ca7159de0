"""CPU oracle of meshing an edited scene -- TEST INFRASTRUCTURE ONLY (the product package never imports it).

Restates DESIGN.md, "Meshing an edited scene" in numpy, one rounding per operation (numpy arrays neither contract nor widen):
  sweep point  p: the sweep's fp32 grid point (linspace(-1, 1, dim) as torch evaluates it, scaled by extents / 2, [R | t] summed
               left to right, then (x, y, z) -> (x, -z, y));
  target       t = fp32(((T_a0 p0 + T_a1 p1) + T_a2 p2) + T_a3), in fp64 from the fp32 p;
  in box       u = inv (t - b) in fp64, ((inv_a0 d0 + inv_a1 d1) + inv_a2 d2), lo_a <= rint(u_a) <= hi_a; inv and b are the
               grid's index map, inv = diag((dim - 1) / extents) adj(R) / det(R) S^T, b = S (t - R extents / 2);
  take         in box && label(t) == mv && (occ(t) > level || occ_p <= level) && (no piece || the piece keeps t):
               (occ_p, label_p) = (occ(t), mv);
  vacate       otherwise label_p == mv && occ_p > level && (p in the piece || rest drop): occ_p = 0.
The network at t is a callback `evaluate(t) -> (occ, label)`: the caller gives the unedited grid for targets on grid points,
or the fp64 network.  The vertex rule: the label of the nearest solid grid point closer than 2, ties to the lowest linear
index, squared distances ((dx^2 + dy^2) + dz^2) in fp64."""
import numpy as np

from oracle import region_oracle as RO

EMPTY_BOX = (1, 0, 1, 0, 1, 0)
S = np.array([[1.0, 0.0, 0.0], [0.0, 0.0, -1.0], [0.0, 1.0, 0.0]])


def linspace_m11(dim):
    """torch.linspace(-1, 1, dim) in fp32 (start + step i below the half, end - step (dim - 1 - i) above it, one rounding)."""
    step = np.float32(2.0) / np.float32(dim - 1)
    i = np.arange(dim, dtype=np.float64)
    lo = np.float64(step) * i - 1.0                                  # exact in fp64: the fused multiply-add, rounded once
    hi = -np.float64(step) * (dim - 1 - i) + 1.0
    return np.where(np.arange(dim) < dim // 2, lo, hi).astype(np.float32)


def sweep_points(T, extents, dim):
    """The sweep's fp32 grid points [dim^3, 3], C order of (i, j, k)."""
    f = np.float32
    T = np.asarray(T, dtype=np.float64)
    r = T[:3].astype(f)
    s = (np.asarray(extents, dtype=np.float64) / 2.0).astype(f)
    lin = linspace_m11(dim)
    I, J, K = np.meshgrid(np.arange(dim), np.arange(dim), np.arange(dim), indexing="ij")
    q = [lin[X.reshape(-1)] * s[a] for a, X in enumerate((I, J, K))]
    w = [((r[a, 0] * q[0] + r[a, 1] * q[1]) + r[a, 2] * q[2]) + r[a, 3] for a in range(3)]
    return np.stack([w[0], -w[2], w[1]], -1).astype(f)


def grid_index_map(T, extents, dim):
    """(inv [3, 3], b [3]) in fp64: index u = inv (x - b) of a network-frame point x, the kernels' expression."""
    T = np.asarray(T, dtype=np.float64)
    ext = np.asarray(extents, dtype=np.float64)
    R = T[:3, :3]
    adj = np.zeros((3, 3))
    for i in range(3):
        for j in range(3):
            i1, i2, j1, j2 = (j + 1) % 3, (j + 2) % 3, (i + 1) % 3, (i + 2) % 3
            adj[i, j] = R[i1, j1] * R[i2, j2] - R[i1, j2] * R[i2, j1]
    det = (R[0, 0] * adj[0, 0] + R[0, 1] * adj[1, 0]) + R[0, 2] * adj[2, 0]
    w = np.array([T[r, 3] - ((R[r, 0] * (ext[0] / 2.0) + R[r, 1] * (ext[1] / 2.0)) + R[r, 2] * (ext[2] / 2.0)) for r in range(3)])
    b = np.array([w[0], -w[2], w[1]])
    inv = np.zeros((3, 3))
    for a in range(3):
        scale = float(dim - 1) / ext[a]
        ri = adj[a] / det
        inv[a] = [scale * ri[0], scale * -ri[2], scale * ri[1]]
    return inv, b


def targets(trans, pts):
    """t = fp32(trans p) [n, 3], fp64 in the kernels' order."""
    m = np.asarray(trans, dtype=np.float64)
    p = np.asarray(pts, dtype=np.float32).astype(np.float64)
    return np.stack([(((m[a, 0] * p[:, 0] + m[a, 1] * p[:, 1]) + m[a, 2] * p[:, 2]) + m[a, 3]) for a in range(3)],
                    -1).astype(np.float32)


def index_of(inv, b, t):
    """u = inv (t - b) [n, 3] in fp64, the kernels' order."""
    d = np.asarray(t, dtype=np.float32).astype(np.float64) - b[None, :]
    return np.stack([(inv[a, 0] * d[:, 0] + inv[a, 1] * d[:, 1]) + inv[a, 2] * d[:, 2] for a in range(3)], -1)


def in_box(u, box):
    if tuple(int(v) for v in box) == EMPTY_BOX:
        return np.zeros(u.shape[0], dtype=bool)
    lo = np.asarray(box[0::2], dtype=np.float64)
    hi = np.asarray(box[1::2], dtype=np.float64)
    r = np.rint(u)                                                   # half to even, as the kernel's rint
    return np.all((r >= lo) & (r <= hi), axis=-1)


class Piece:
    """A move's piece for the oracle: region words, dim, voxel map and outside policy, for a label it applies to."""

    def __init__(self, bits, dim, vmap, outside_keep):
        self.bits, self.dim, self.vmap, self.outside_keep = np.asarray(bits).view(np.uint32), int(dim), vmap, bool(outside_keep)

    def keeps(self, pts):
        b = RO.lookup(self.vmap, self.bits, self.dim, pts)
        return (b == 1) | ((b < 0) & self.outside_keep)


def solid_box(occ, labels, label, level, margin, keep=None):
    """objects.solid_box on numpy grids."""
    mask = (labels == label) & (occ > np.float32(level))
    if keep is not None:
        mask &= keep
    if not mask.any():
        return EMPTY_BOX
    dim = occ.shape[0]
    out = []
    for a in range(3):
        idx = np.nonzero(mask.any(axis=tuple(c for c in range(3) if c != a)))[0]
        out += [max(int(idx[0]) - margin, 0), min(int(idx[-1]) + margin, dim - 1)]
    return tuple(out)


def apply_move(occ, labels, pts, inv, b, move, evaluate, level):
    """One move on flat grids occ [n] float32, labels [n] int (edited in place) -> number of targets evaluated.
    move: dict(label, trans 4x4 (or 3x4), box, piece (Piece or None), rest_drop)."""
    mv, piece = int(move["label"]), move.get("piece")
    lev = np.float32(level)
    t = targets(np.asarray(move["trans"], dtype=np.float64)[:3], pts)
    inb = in_box(index_of(inv, b, t), move["box"])
    idx = np.nonzero(inb)[0]
    take = np.zeros(occ.shape[0], dtype=bool)
    occ_t = np.zeros(occ.shape[0], dtype=np.float32)
    if idx.size:
        o_t, l_t = evaluate(t[idx])
        occ_t[idx] = o_t
        ok = (np.asarray(l_t) == mv) & ((np.asarray(o_t) > lev) | (occ[idx] <= lev))
        if piece is not None:
            ok &= piece.keeps(t[idx])
        take[idx] = ok
    in_piece = np.ones(occ.shape[0], dtype=bool) if piece is None else piece.keeps(pts)
    vacate = ~take & (labels == mv) & (occ > lev) & (in_piece | bool(move.get("rest_drop", False)))
    occ[take] = occ_t[take]
    labels[take] = mv
    occ[vacate] = 0.0
    return int(idx.size)


def edit(occ, labels, T, extents, moves, evaluate, level):
    """The moves applied in order to copies of occ / labels [dim]^3 -> (occ, labels, evaluated)."""
    dim = occ.shape[0]
    o, lab = occ.reshape(-1).astype(np.float32).copy(), labels.reshape(-1).astype(np.int64).copy()
    pts = sweep_points(T, extents, dim)
    inv, b = grid_index_map(T, extents, dim)
    n = 0
    for mv in moves:
        n += apply_move(o, lab, pts, inv, b, mv, evaluate, level)
    return o.reshape(occ.shape), lab.reshape(occ.shape).astype(labels.dtype), n


def grid_evaluate(occ, labels, inv, b):
    """evaluate() for targets on grid points: the unedited grid at rint(u); a target off the grid points raises."""
    dim = occ.shape[0]

    def f(t):
        u = index_of(inv, b, t)
        i = np.rint(u)
        assert np.array_equal(i, u), "a target is not on a grid point"
        assert ((i >= 0) & (i <= dim - 1)).all(), "a target is outside the grid"
        ii = i.astype(np.int64)
        return occ[ii[:, 0], ii[:, 1], ii[:, 2]], labels[ii[:, 0], ii[:, 1], ii[:, 2]]
    return f


def vertex_labels(verts, occ, labels, level):
    """The label of the nearest solid grid point closer than 2 per index-space vertex [n, 3] (ties: lowest linear index; -1:
    none) -> int64 [n]."""
    dim = occ.shape[0]
    v = np.asarray(verts, dtype=np.float32).reshape(-1, 3)
    solid = occ > np.float32(level)
    out = np.full(v.shape[0], -1, dtype=np.int64)
    for q in range(v.shape[0]):
        x = v[q].astype(np.float64)
        if not (np.isfinite(x).all() and (x > -2).all() and (x < dim + 1).all()):
            continue
        f = np.floor(x).astype(np.int64)
        best, bd = -1, 4.0
        for i in range(max(f[0] - 1, 0), min(f[0] + 2, dim - 1) + 1):
            dx = x[0] - i
            for j in range(max(f[1] - 1, 0), min(f[1] + 2, dim - 1) + 1):
                dy = x[1] - j
                dxy = dx * dx + dy * dy
                for k in range(max(f[2] - 1, 0), min(f[2] + 2, dim - 1) + 1):
                    dz = x[2] - k
                    d2 = dxy + dz * dz
                    if d2 < bd and solid[i, j, k]:
                        bd, best = d2, int(labels[i, j, k])
        out[q] = best
    return out


def nearest_solid_bruteforce(verts, occ, labels, level):
    """The same rule by a search over every solid point of the grid (for small grids): the independent check of the block walk."""
    dim = occ.shape[0]
    idx = np.argwhere(occ > np.float32(level))                      # ascending linear index
    out = np.full(len(verts), -1, dtype=np.int64)
    for q, x in enumerate(np.asarray(verts, dtype=np.float32).astype(np.float64)):
        if not len(idx):
            continue
        d = idx.astype(np.float64) - x[None, :]
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        k = int(np.argmin(d2))                                       # first minimum = lowest linear index
        if d2[k] < 4.0:
            out[q] = int(labels[tuple(idx[k])])
    return out
