"""CPU oracle of the object inventory -- TEST INFRASTRUCTURE ONLY (the product package never imports it).

Restates every definition of DESIGN.md, "Object inventory", point by point on the grid with np.nonzero, in int64 / fp64:
a grid point is solid when occ > level (level held in float32, as the kernels compare it); a group is one label (no label grid:
one group); trimming keeps, per axis, the sorted coordinates from position floor(trim N) to N - 1 - floor(trim N); an object's
points are its solid points inside that box, and every statistic is taken over them, each point mapped to the network frame on
its own (linspace, extents / 2, [R | t], then (x, y, z) -> (x, -z, y))."""
import numpy as np


def index_to_network(idx, T, dim, extents):
    """Grid indices [n, 3] -> network-frame points [n, 3] in fp64, one point at a time (no matrix form)."""
    idx = np.asarray(idx, dtype=np.float64).reshape(-1, 3)
    T = np.asarray(T, dtype=np.float64)
    ext = np.asarray(extents, dtype=np.float64)
    q = (-1.0 + 2.0 * idx / (dim - 1)) * (ext / 2.0)
    w = q @ T[:3, :3].T + T[:3, 3]
    return np.stack([w[:, 0], -w[:, 2], w[:, 1]], -1)


def grid_points_fp32(idx, T, dim, extents):
    """numpy twin of grid_points_kernel's fp32 arithmetic (mesh.cu): the sweep's own grid points for indices [n, 3]."""
    idx = np.asarray(idx, dtype=np.int64).reshape(-1, 3)
    f = np.float32
    step = f(2.0) / f(dim - 1)
    r = np.asarray(T, dtype=np.float64)[:3].astype(f)
    s = (np.asarray(extents, dtype=np.float64) / 2.0).astype(f)

    def lin(i):                                          # fma in fp32 = exact fp64 product and sum, rounded once
        lo = (np.float64(step) * i.astype(np.float64) - 1.0).astype(f)
        hi = (-np.float64(step) * (dim - 1 - i).astype(np.float64) + 1.0).astype(f)
        return np.where(i < dim // 2, lo, hi)
    q = [lin(idx[:, a]) * s[a] for a in range(3)]
    w = [((r[row, 0] * q[0] + r[row, 1] * q[1]) + r[row, 2] * q[2]) + r[row, 3] for row in range(3)]
    return np.stack([w[0], -w[2], w[1]], -1).astype(f)


def group_points(occ, labels, level, g):
    """Indices [n, 3] int64 of the solid points of group g."""
    solid = np.asarray(occ) > np.float32(level)
    if labels is not None:
        solid &= np.asarray(labels) == g
    return np.stack(np.nonzero(solid), -1).astype(np.int64)


def moments(idx):
    """count, Si, Sj, Sk, Sii, Sjj, Skk, Sij, Sik, Sjk (int64) of indices [n, 3]."""
    i, j, k = idx[:, 0], idx[:, 1], idx[:, 2]
    return np.array([idx.shape[0], i.sum(), j.sum(), k.sum(), (i * i).sum(), (j * j).sum(), (k * k).sum(), (i * j).sum(),
                     (i * k).sum(), (j * k).sum()], dtype=np.int64)


def histograms(idx, dim):
    return np.stack([np.bincount(idx[:, a], minlength=dim) for a in range(3)]).astype(np.uint32)


def trimmed_box(idx, trim):
    """(i_lo, i_hi, j_lo, j_hi, k_lo, k_hi): per axis the sorted coordinates at floor(trim N) and N - 1 - floor(trim N)."""
    n = idx.shape[0]
    cut = int(np.floor(trim * n))
    out = []
    for a in range(3):
        s = np.sort(idx[:, a])
        out += [int(s[cut]), int(s[n - 1 - cut])]
    return np.array(out, dtype=np.int32)


def in_box(idx, box):
    keep = np.ones(idx.shape[0], dtype=bool)
    for a in range(3):
        keep &= (idx[:, a] >= box[2 * a]) & (idx[:, a] <= box[2 * a + 1])
    return idx[keep]


def obb_axes(cov):
    """Rows: eigenvectors of cov, descending eigenvalue, largest-magnitude component positive, third = first x second."""
    w, V = np.linalg.eigh(cov)
    axes = V[:, ::-1].T.copy()
    for r in range(2):
        if axes[r, np.argmax(np.abs(axes[r]))] < 0:
            axes[r] = -axes[r]
    axes[2] = np.cross(axes[0], axes[1])
    return axes


def inventory(occ, labels, T, extents, level=0.45, trim=0.0, n_labels=None):
    """{label: entry} of every group with points: the integer statistics (moments, hist of the solid points; object_moments
    of the object's points), box, voxels, volume, centre, covariance, aabb and the OBB (axes, centre, half_sizes)."""
    occ = np.asarray(occ)
    dim = occ.shape[0]
    T = np.asarray(T, dtype=np.float64)
    ext = np.asarray(extents, dtype=np.float64)
    n_labels = (128 if labels is not None else 1) if n_labels is None else n_labels
    out = {}
    for g in range(n_labels):
        idx = group_points(occ, labels, level, g)
        if idx.shape[0] == 0:
            continue
        box = trimmed_box(idx, trim)
        obj = in_box(idx, box)
        e = {"moments": moments(idx), "hist": histograms(idx, dim), "box": box, "object_moments": moments(obj),
             "voxels": obj.shape[0]}
        if obj.shape[0]:
            p = index_to_network(obj, T, dim, extents)
            centre = p.mean(0)
            cov = (p - centre).T @ (p - centre) / p.shape[0]
            corners = np.array([[box[2 * a + ((c >> a) & 1)] for a in range(3)] for c in range(8)])
            q = index_to_network(corners, T, dim, extents)
            axes = obb_axes(cov)
            proj = (p - centre) @ axes.T
            lo, hi = proj.min(0), proj.max(0)
            e.update(volume=obj.shape[0] * abs(np.linalg.det(T[:3, :3])) * np.prod(ext / (dim - 1)), centre=centre, covariance=cov,
                     aabb=(q.min(0), q.max(0)), obb={"axes": axes, "centre": centre + axes.T @ ((lo + hi) / 2),
                                                    "half_sizes": (hi - lo) / 2})
        out[g] = e
    return out


def project(occ, labels, level, g, box, axes_row):
    """min, max of ((u0 i + u1 j) + u2 k) + o over group g's points in box: the spans pass's formula, operation by operation."""
    idx = in_box(group_points(occ, labels, level, g), box).astype(np.float64)
    u0, u1, u2, o = axes_row
    s = ((u0 * idx[:, 0] + u1 * idx[:, 1]) + u2 * idx[:, 2]) + o
    return (s.min(), s.max()) if s.size else (np.inf, -np.inf)
