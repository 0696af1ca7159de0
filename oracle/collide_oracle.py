"""CPU oracle of the collision checks -- TEST INFRASTRUCTURE ONLY (the product package never imports it).

Restates DESIGN.md, "Collision checks" in numpy, one rounding per fp64 operation, on top of edit_sweep_oracle's sweep points,
index map, targets, nearest indices, boxes and pieces:
  src(p)       q = rint(inv (t - b)) of t = fp32(trans p) in the source box B, labels[q] == mv, occ[q] > level and (no piece or the
               piece keeps t): the moved object covers p;
  obstacle(p)  occ[p] > level and labels[p] in the obstacle labels, unless labels[p] == mv and (p in the piece -- every point
               without a piece -- or rest dropped);
  landed       #{p : src(p)};  overlap[l] = #{p : src(p) and obstacle(p) and labels[p] == l};
  faces[a, l1, l2] = #{p : solid l1 at p, solid l2 at p + e_a, l1 != l2}.
destination_box restates the culling: the index box every p with src(p) lies in."""
import numpy as np

from oracle import edit_sweep_oracle as E

N_LABELS = 128


def destination_box(T, extents, dim, trans, box):
    """(lo [3], hi [3]) int of the grid points that can land in `box` under `trans`, or None: B grown by half a voxel, its
    corners mapped by idx_p = A^-1 (trans^-1 (A u + b) - b), floor / ceil, one voxel of margin, clipped to the grid."""
    if tuple(int(v) for v in box) == E.EMPTY_BOX:
        return None
    inv, b = E.grid_index_map(T, extents, dim)
    A = np.linalg.inv(inv)
    m = np.asarray(trans, dtype=np.float64)
    Mi = np.linalg.inv(m[:3, :3])
    lo, hi = np.asarray(box[0::2], dtype=np.float64) - 0.5, np.asarray(box[1::2], dtype=np.float64) + 0.5
    corners = np.array([[(hi if (c >> a) & 1 else lo)[a] for a in range(3)] for c in range(8)])
    v = ((corners @ A.T + b - m[:3, 3]) @ Mi.T - b) @ inv.T
    if not np.isfinite(v).all():
        return np.zeros(3, dtype=np.int64), np.full(3, dim - 1, dtype=np.int64)
    dlo = np.clip(np.floor(v.min(0)) - 1, 0, dim).astype(np.int64)
    dhi = np.clip(np.ceil(v.max(0)) + 1, -1, dim - 1).astype(np.int64)
    return (dlo, dhi) if (dlo <= dhi).all() else None


def move_overlap(occ, labels, T, extents, moves, level, obstacles=None, cull=True):
    """Each move (dict: label, trans 4x4, box, piece (E.Piece or None), rest_drop) on its own against occ / labels [dim]^3 ->
    (overlap int64 [n, 128], landed int64 [n]).  obstacles: the obstacle labels (None: every label).  cull: visit only each
    move's destination box (the kernel's work), else the whole grid; the counts must not differ."""
    dim = occ.shape[0]
    o, lab = occ.reshape(-1).astype(np.float32), labels.reshape(-1).astype(np.int64)
    lev = np.float32(level)
    pts = E.sweep_points(T, extents, dim)
    inv, b = E.grid_index_map(T, extents, dim)
    is_obst = np.ones(N_LABELS, dtype=bool) if obstacles is None else np.isin(np.arange(N_LABELS), list(obstacles))
    solid = o > lev
    blocking = solid & is_obst[np.clip(lab, 0, N_LABELS - 1)]
    idx = np.stack(np.meshgrid(*[np.arange(dim)] * 3, indexing="ij"), -1).reshape(-1, 3)
    overlap = np.zeros((len(moves), N_LABELS), dtype=np.int64)
    landed = np.zeros(len(moves), dtype=np.int64)
    for i, mv in enumerate(moves):
        label, piece = int(mv["label"]), mv.get("piece")
        visit = np.ones(o.shape[0], dtype=bool)
        if cull:
            box = destination_box(T, extents, dim, mv["trans"], mv["box"])
            if box is None:
                continue
            visit = np.all((idx >= box[0]) & (idx <= box[1]), axis=1)
        sel = np.nonzero(visit)[0]
        t = E.targets(np.asarray(mv["trans"], dtype=np.float64)[:3], pts[sel])
        u = E.index_of(inv, b, t)
        src = E.in_box(u, mv["box"])
        q = np.rint(u[src]).astype(np.int64)
        qi = (q[:, 0] * dim + q[:, 1]) * dim + q[:, 2]
        ok = (lab[qi] == label) & (o[qi] > lev)
        if piece is not None:
            ok &= piece.keeps(t[src])
        src[np.nonzero(src)[0]] = ok
        p = sel[src]
        landed[i] = p.size
        vacated = lab[p] == label
        if piece is not None and not mv.get("rest_drop", False):
            vacated &= piece.keeps(pts[p])
        hit = p[blocking[p] & ~vacated]
        overlap[i] = np.bincount(lab[hit], minlength=N_LABELS)
    return overlap, landed


def object_contacts(occ, labels, level, n_labels=N_LABELS):
    """faces int64 [3, n_labels, n_labels] of a labelled grid."""
    solid = occ > np.float32(level)
    lab = labels.astype(np.int64)
    faces = np.zeros((3, n_labels, n_labels), dtype=np.int64)
    for a in range(3):
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[a], hi[a] = slice(0, -1), slice(1, None)
        l1, l2 = lab[tuple(lo)], lab[tuple(hi)]
        both = solid[tuple(lo)] & solid[tuple(hi)] & (l1 != l2)
        np.add.at(faces[a], (l1[both], l2[both]), 1)
    return faces
