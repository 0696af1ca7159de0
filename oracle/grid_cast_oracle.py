"""CPU oracle of casting rays through a labelled grid -- TEST INFRASTRUCTURE ONLY (the product package never imports it).

Restates DESIGN.md, "Viewing the labelled grid" in numpy, one rounding per fp64 operation (numpy arrays neither contract nor
widen), as the voxel-by-voxel walk the kernel takes:
  index space  u(t) = u0 + t w, u0 = inv (o - b) and w = inv d, inv and b the grid's index map (edit_sweep_oracle.grid_index_map),
               each row ((inv_a0 x0 + inv_a1 x1) + inv_a2 x2);
  clip         t in [near, far] and in the grid's cube [-1/2, dim - 1/2]^3: per axis with w_a != 0 the times (lo - u0_a) / w_a and
               (hi - u0_a) / w_a (lo / hi swapped for w_a < 0); an axis with w_a == 0 must have u0_a in [lo, hi]; t0 = max(near,
               entry), t1 = min(far, exit), a miss unless t0 <= t1;
  start        q = clamp(floor((u0 + t0 w) + 1/2), 0, dim - 1);
  step         the next boundary time of axis a is (q_a + s_a / 2 - u0_a) / w_a, s_a = sign w_a; the smallest one is stepped, ties
               i before j before k; the walk stops (a miss) when that time exceeds t1 or q leaves the grid;
  hit          occ[q] > level and, under a keep mask, the label in [0, 127] and kept: t = fp32(max(t0, t_entry) + 0), the label and
               the C-order index of q;
  normal       -inv^T g normalised, g the central difference of occ at q (one-sided at the grid's faces); where g gives zero or a
               non-finite length, the entry face's normal inv^T (-s_a e_a), or -d for a ray that starts inside the voxel.  The
               normals are returned in float64: the kernel's float32 normals are held to a tolerance."""
import numpy as np

from oracle import edit_sweep_oracle as E


def _kept(labels, keep_words):
    if keep_words is None:
        return np.ones(labels.shape, dtype=bool)
    l = labels.astype(np.int64)
    words = np.asarray(keep_words, dtype=np.uint64)
    inside = (l >= 0) & (l <= 127)
    lc = np.clip(l, 0, 127)
    return inside & (((words[lc >> 5] >> (lc & 31).astype(np.uint64)) & np.uint64(1)) == 1)


def _rows(inv, x):
    """inv x per row in the kernel's order, x [n, 3] float64."""
    return np.stack([(inv[a, 0] * x[:, 0] + inv[a, 1] * x[:, 1]) + inv[a, 2] * x[:, 2] for a in range(3)], -1)


def _normal(inv, g):
    n = -np.stack([(inv[0, c] * g[:, 0] + inv[1, c] * g[:, 1]) + inv[2, c] * g[:, 2] for c in range(3)], -1)
    return n, (n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2]


def cast(occ, labels, T, extents, rays_o, rays_d, near, far, level=0.45, keep_words=None):
    """The flat walk of every ray -> dict(t float32 [n] (+inf: no hit), label int16 [n], voxel int32 [n] (-1: no hit),
    normal float64 [n, 3] (0: no hit), start_inside bool [n])."""
    occ = np.asarray(occ, dtype=np.float32)
    labels = np.asarray(labels)
    dim = occ.shape[0]
    occ_f, lab_f = occ.reshape(-1), labels.reshape(-1)
    inv, b = E.grid_index_map(T, extents, dim)
    o = np.asarray(rays_o, dtype=np.float32).reshape(-1, 3)
    d = np.asarray(rays_d, dtype=np.float32).reshape(-1, 3)
    n = o.shape[0]
    lev = np.float32(level)
    near, far = float(np.float32(near)), float(np.float32(far))
    with np.errstate(all="ignore"):
        u0 = _rows(inv, o.astype(np.float64) - b[None, :])
        w = _rows(inv, d.astype(np.float64))
        ok = np.isfinite(u0).all(1) & np.isfinite(w).all(1) & (w != 0).any(1)
        lo, hi = -0.5, dim - 0.5
        s = np.where(w > 0, 1, -1)
        t_in = np.full(n, -np.inf)
        in_axis = np.full(n, -1)
        t_exit = np.full(n, np.inf)
        for a in range(3):
            moving = w[:, a] != 0
            ok &= moving | ((u0[:, a] >= lo) & (u0[:, a] <= hi))
            ta = (np.where(s[:, a] > 0, lo, hi) - u0[:, a]) / w[:, a]
            tb = (np.where(s[:, a] > 0, hi, lo) - u0[:, a]) / w[:, a]
            upd = moving & (ta > t_in)
            t_in = np.where(upd, ta, t_in)
            in_axis = np.where(upd, a, in_axis)
            t_exit = np.where(moving, np.fmin(t_exit, tb), t_exit)
        t0 = np.fmax(near, t_in)
        t1 = np.fmin(far, t_exit)
        ok &= t0 <= t1
        q = np.clip(np.floor((u0 + t0[:, None] * w) + 0.5), 0, dim - 1)
        q = np.where(np.isfinite(q), q, 0).astype(np.int64)

        def boundary(qa, a):
            return ((qa + 0.5 * s[:, a]) - u0[:, a]) / w[:, a]
        tn = np.stack([np.where(w[:, a] != 0, boundary(q[:, a], a), np.inf) for a in range(3)], -1)
    t_entry = t0.copy()
    e_axis = np.where(t_in >= near, in_axis, -1)
    t_out = np.full(n, np.inf, dtype=np.float32)
    label = np.full(n, -1, dtype=np.int16)
    voxel = np.full(n, -1, dtype=np.int32)
    hit_axis = np.full(n, -1)
    active = ok.copy()
    for _ in range(3 * dim + 3):
        idx = np.nonzero(active)[0]
        if not idx.size:
            break
        p = (q[idx, 0] * dim + q[idx, 1]) * dim + q[idx, 2]
        solid = (occ_f[p] > lev) & _kept(lab_f[p], keep_words)
        h = idx[solid]
        t_out[h] = (np.maximum(t0[h], t_entry[h]) + 0.0).astype(np.float32)   # + 0: a zero time is +0
        label[h] = lab_f[p[solid]]
        voxel[h] = p[solid]
        hit_axis[h] = e_axis[h]
        active[h] = False
        m = idx[~solid]
        tm = tn[m]
        a = np.where(tm[:, 1] < tm[:, 0], 1, 0)
        ta = tm[np.arange(m.size), a]
        a = np.where(tm[:, 2] < ta, 2, a)
        ta = tm[np.arange(m.size), a]
        go = ta <= t1[m]
        active[m[~go]] = False
        m, a, ta = m[go], a[go], ta[go]
        q[m, a] += s[m, a]
        inside = (q[m, a] >= 0) & (q[m, a] < dim)
        active[m[~inside]] = False
        m, a, ta = m[inside], a[inside], ta[inside]
        t_entry[m] = ta
        e_axis[m] = a
        with np.errstate(all="ignore"):
            tn[m, a] = ((q[m, a] + 0.5 * s[m, a]) - u0[m, a]) / w[m, a]
    normal = np.zeros((n, 3))
    h = np.nonzero(voxel >= 0)[0]
    if h.size:
        occ64 = occ.astype(np.float64)
        qh = np.stack(np.unravel_index(voxel[h].astype(np.int64), occ.shape), -1)
        g = np.zeros((h.size, 3))
        for a in range(3):
            up, dn = qh.copy(), qh.copy()
            has_hi, has_lo = qh[:, a] < dim - 1, qh[:, a] > 0
            up[:, a] = np.where(has_hi, qh[:, a] + 1, qh[:, a])
            dn[:, a] = np.where(has_lo, qh[:, a] - 1, qh[:, a])
            diff = occ64[tuple(up.T)] - occ64[tuple(dn.T)]
            g[:, a] = np.where(has_hi & has_lo, diff * 0.5, diff)
        with np.errstate(all="ignore"):
            nv, nn = _normal(inv, g)
            bad = ~(nn > 0) | ~np.isfinite(nn)
            ea = hit_axis[h]
            face = np.zeros((h.size, 3))
            face[np.arange(h.size), np.clip(ea, 0, 2)] = s[h, np.clip(ea, 0, 2)]
            fv, fn = _normal(inv, face)
            dv = -d[h].astype(np.float64)
            dn2 = (dv[:, 0] * dv[:, 0] + dv[:, 1] * dv[:, 1]) + dv[:, 2] * dv[:, 2]
            nv = np.where(bad[:, None], np.where((ea >= 0)[:, None], fv, dv), nv)
            nn = np.where(bad, np.where(ea >= 0, fn, dn2), nn)
            normal[h] = nv * (1.0 / np.sqrt(nn))[:, None]
    return dict(t=t_out, label=label, voxel=voxel, normal=normal, start_inside=(hit_axis < 0) & (voxel >= 0))
