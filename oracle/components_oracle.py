"""CPU oracle of the connected components -- TEST INFRASTRUCTURE ONLY (the product package never imports it).

Restates DESIGN.md, "Connected components", with scipy.ndimage.label: a grid point is solid when occ > level (level held in
float32, as the kernels compare it); per label k the components of solid & (labels == k) under face neighbours
(generate_binary_structure(3, 1), connectivity 6) or all 26 neighbours (np.ones((3, 3, 3))), which never wrap across a grid
face; then every component numbered by its smallest C-order linear index, ascending.  Also the hand-made grids the tests and
tools/components_bench.py share."""
import numpy as np
from scipy import ndimage


def components(occ, labels=None, level=0.45, connectivity=26):
    """-> (grid int32 [dim]^3: id or -1, label int16 [n], voxels int64 [n], root int64 [n])."""
    occ = np.asarray(occ)
    if connectivity not in (6, 26):
        raise ValueError("connectivity %r is not 6 or 26" % (connectivity,))
    structure = ndimage.generate_binary_structure(3, 1) if connectivity == 6 else np.ones((3, 3, 3), dtype=bool)
    solid = occ > np.float32(level)
    labels = np.zeros(occ.shape, dtype=np.int16) if labels is None else np.asarray(labels)
    parts = []                                   # per label: (k, flat indices, their local ids 0 .., roots of the local ids)
    for k in np.unique(labels[solid]):
        lab, _ = ndimage.label(solid & (labels == k), structure=structure)
        flat = lab.reshape(-1)
        idx = np.nonzero(flat)[0]
        local = flat[idx].astype(np.int64) - 1
        _, first = np.unique(local, return_index=True)          # indices ascend: the first point of a component is its root
        parts.append((int(k), idx, local, idx[first]))
    roots = np.concatenate([p[3] for p in parts]) if parts else np.zeros(0, np.int64)
    labs = np.concatenate([np.full(p[3].size, p[0], np.int16) for p in parts]) if parts else np.zeros(0, np.int16)
    order = np.argsort(roots, kind="stable")
    gid = np.empty(order.size, np.int64)
    gid[order] = np.arange(order.size)
    grid = np.full(occ.size, -1, dtype=np.int32)
    at = 0
    for _, idx, local, r in parts:
        grid[idx] = gid[at + local]
        at += r.size
    voxels = np.bincount(grid[grid >= 0], minlength=order.size).astype(np.int64)
    return grid.reshape(occ.shape), labs[order], voxels, roots[order].astype(np.int64)


def largest(label, voxels, root):
    """{label: component id with the most voxels, the smaller root on a tie}."""
    best = {}
    for c in range(len(label)):
        k = int(label[c])
        if k not in best or (voxels[c], -root[c]) > (voxels[best[k]], -root[best[k]]):
            best[k] = c
    return best


# ---- hand-made grids ---------------------------------------------------------------------------------------------------------
def serpentine(dim):
    """occ [dim]^3 float32 (1 solid, 0 not) holding one path through the grid: in every even i-plane the even j-rows, joined at
    alternate ends through the odd rows; consecutive even planes joined through one point of the odd plane between them, at
    alternate ends of the plane's path.  One component under 6- and 26-connectivity."""
    occ = np.zeros((dim,) * 3, np.float32)
    rows = list(range(0, dim, 2))
    ends = [(0, 0), (rows[-1], dim - 1 if (len(rows) - 1) % 2 == 0 else 0)]    # a plane's path starts at one, ends at the other
    for i in range(0, dim, 2):
        for r, j in enumerate(rows):
            occ[i, j, :] = 1
            if j + 2 < dim:
                occ[i, j + 1, dim - 1 if r % 2 == 0 else 0] = 1
        if i + 2 < dim:
            j, k = ends[1 - (i // 2) % 2]
            occ[i + 1, j, k] = 1
    return occ


def checkerboard(dim):
    """occ [dim]^3 float32: solid where i + j + k is even.  Every point its own component under 6, one component under 26."""
    i, j, k = np.meshgrid(*[np.arange(dim)] * 3, indexing="ij")
    return ((i + j + k) % 2 == 0).astype(np.float32)
