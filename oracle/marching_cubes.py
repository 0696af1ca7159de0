"""Table-free marching cubes in numpy -- TEST INFRASTRUCTURE ONLY: the cross-check of the case table the library generates
(dm-nerf_b200/csrc/mesh.cu).  Every cell is polygonised by walking its six faces; nothing is looked up.

Conventions (DESIGN.md, "Mesh extraction"):
  * inside = value > level; NaN is never inside (the library rejects a grid holding NaN before it gets here).
  * one vertex per grid edge whose endpoints differ in inside-ness, at p0 + t along the edge's axis in index units,
    t = (level - v0) / (v1 - v0) in float32 (v0 at the lower index), position = float32(index) + t.
  * vertices are numbered by global edge id 3 * (flat C-order index of the edge's lower point) + axis.
  * face ambiguity: a face whose inside corners are diagonal keeps them separate (each gets its own segment).
  * winding: face normals point toward increasing value (toward the inside).
  * triangles: cells in C order of their lowest corner; inside a cell the loops in order of their smallest local edge, each walked
    in the oriented direction from that edge and cut into a fan from its first vertex none of whose chords joins two edges of
    one face (such a chord would lie in the face, shared with the neighbouring cell's fan).
"""
import numpy as np

# corner c of a cell: bit a = offset along axis a.  Local edge e = 4 * axis + r, r = the two other axes' bits (lower axis first).
_OTHER = {0: (1, 2), 1: (0, 2), 2: (0, 1)}


def _edge_corners(e):
    a, r = divmod(e, 4)
    b, c = _OTHER[a]
    lo = ((r & 1) << b) | ((r >> 1) << c)
    return lo, lo | (1 << a)


def _pos2(c):
    """Corner position, doubled (integer)."""
    return np.array([(c >> 0) & 1, (c >> 1) & 1, (c >> 2) & 1]) * 2


def _mid2(e):
    lo, hi = _edge_corners(e)
    return (_pos2(lo) + _pos2(hi)) // 2


def _face_segments(inside, a, s):
    """Directed segments (from edge, to edge) of face (axis a, side s) of a cell with corner inside-ness `inside` [8]."""
    corners = [c for c in range(8) if ((c >> a) & 1) == s]
    edges = [e for e in range(12) if e // 4 != a and ((_edge_corners(e)[0] >> a) & 1) == s]
    cross = [e for e in edges if inside[_edge_corners(e)[0]] != inside[_edge_corners(e)[1]]]
    n_face = np.zeros(3, dtype=np.int64)
    n_face[a] = 1 if s else -1
    pairs = []
    if len(cross) == 2:
        ins = [c for c in corners if inside[c]]
        # from the segment's midpoint toward the centroid of the face's inside corners (times 4 len(ins))
        toward = 2 * sum(_pos2(c) for c in ins) - len(ins) * (_mid2(cross[0]) + _mid2(cross[1]))
        pairs.append((cross[0], cross[1], toward))
    elif len(cross) == 4:
        for c in corners:
            if inside[c]:
                mine = [e for e in cross if c in _edge_corners(e)]
                toward = 2 * _pos2(c) - (_mid2(mine[0]) + _mid2(mine[1]))
                pairs.append((mine[0], mine[1], toward))
    out = []
    for e0, e1, toward in pairs:
        d = _mid2(e1) - _mid2(e0)
        if np.dot(d, np.cross(n_face, toward)) > 0:
            e0, e1 = e1, e0
        out.append((e0, e1))
    return out


def cell_polygons(inside):
    """Oriented loops (lists of local edges) of one cell, in the library's triangle order."""
    nxt = {}
    for a in range(3):
        for s in range(2):
            for e0, e1 in _face_segments(inside, a, s):
                assert e0 not in nxt, "two segments leave edge %d" % e0
                nxt[e0] = e1
    loops, seen = [], set()
    for e in sorted(nxt):
        if e in seen:
            continue
        loop = [e]
        seen.add(e)
        while nxt[loop[-1]] != e:
            loop.append(nxt[loop[-1]])
            seen.add(loop[-1])
        loops.append(loop)
    return loops


def _faces_of(e):
    lo, _ = _edge_corners(e)
    return {(b, (lo >> b) & 1) for b in range(3) if b != e // 4}


def cell_triangles(inside):
    """Each loop as a fan from its first vertex (in walk order) none of whose chords joins two edges of one face."""
    tris = []
    for loop in cell_polygons(inside):
        n = len(loop)
        apex = next(k for k in range(n)
                    if all(not (_faces_of(loop[k]) & _faces_of(loop[j])) for j in range(n) if j not in (k, (k + 1) % n, (k - 1) % n)))
        for i in range(1, n - 1):
            tris.append((loop[apex], loop[(apex + i) % n], loop[(apex + i + 1) % n]))
    return tris


def marching_cubes(grid, level):
    """grid [nx, ny, nz] -> (verts float32 [V, 3] in index units, tris int64 [T, 3], edge_ids int64 [V])."""
    g = np.asarray(grid, dtype=np.float32)
    lev = np.float32(level)
    assert not np.isnan(g).any(), "NaN in the grid"
    nx, ny, nz = g.shape
    inside = g > lev
    ids, pos = [], []
    for a in range(3):
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[a], hi[a] = slice(0, -1), slice(1, None)
        v0, v1 = g[tuple(lo)], g[tuple(hi)]
        crossing = inside[tuple(lo)] != inside[tuple(hi)]
        idx = np.argwhere(crossing)
        with np.errstate(divide="ignore", invalid="ignore"):
            t = (lev - v0[crossing]) / (v1[crossing] - v0[crossing])
        p = idx.astype(np.float32)
        p[:, a] = p[:, a] + t.astype(np.float32)
        ids.append(3 * ((idx[:, 0] * ny + idx[:, 1]) * nz + idx[:, 2]) + a)
        pos.append(p)
    ids = np.concatenate(ids)
    pos = np.concatenate(pos)
    order = np.argsort(ids, kind="stable")
    ids, pos = ids[order], pos[order]
    vid = {int(e): i for i, e in enumerate(ids)}
    tris = []
    cube = np.zeros((nx - 1, ny - 1, nz - 1), dtype=np.int64)
    for c in range(8):
        cube |= inside[(c & 1):nx - 1 + (c & 1), ((c >> 1) & 1):ny - 1 + ((c >> 1) & 1),
                       ((c >> 2) & 1):nz - 1 + ((c >> 2) & 1)].astype(np.int64) << c
    for i, j, k in np.argwhere((cube != 0) & (cube != 255)):
        case = int(cube[i, j, k])
        ins = [(case >> c) & 1 for c in range(8)]
        for tri in cell_triangles(ins):
            row = []
            for e in tri:
                a = e // 4
                lo, _ = _edge_corners(e)
                p = (i + (lo & 1), j + ((lo >> 1) & 1), k + ((lo >> 2) & 1))
                row.append(vid[3 * ((p[0] * ny + p[1]) * nz + p[2]) + a])
            tris.append(row)
    return pos.astype(np.float32), np.asarray(tris, dtype=np.int64).reshape(-1, 3), ids
