"""CPU oracle of deforming objects -- TEST INFRASTRUCTURE ONLY (the product package never imports it).

Restates DESIGN.md, "Deforming objects" in numpy, fp64 with one rounding per operation (numpy arrays neither contract nor
widen), on top of the edit-sweep, collision, moved-render and group oracles.  A deformed move is a move dict with "deform": any
value with frame [12] (e_u, e_v, e_h, c), h0, dh and knots [K, 6] (A row-major, then t) -- an objects.Deformation qualifies.
The target of a grid point p is x = D^-1(trans p), rounded once to fp32, and every rule (take, vacate, pieces, copies, groups,
boxes) is group_oracle's with that target; a move without "deform" is group_oracle's own move."""
import numpy as np
import torch

from oracle import edit_sweep_oracle as E
from oracle import group_oracle as GO
from oracle import render_moves_oracle as RM

N_LABELS = GO.N_LABELS


def _table(d):
    frame = np.asarray(d.frame if hasattr(d, "frame") else d["frame"], dtype=np.float64).reshape(12)
    get = (lambda k: getattr(d, k)) if hasattr(d, "frame") else (lambda k: d[k])
    return frame, float(get("h0")), float(get("dh")), np.asarray(get("knots"), dtype=np.float64).reshape(-1, 6)


def moved(trans, pts):
    """y = trans p [n, 3] in fp64, the kernels' order, not rounded."""
    m = np.asarray(trans, dtype=np.float64)
    p = np.asarray(pts, dtype=np.float32).astype(np.float64)
    return np.stack([(((m[a, 0] * p[:, 0] + m[a, 1] * p[:, 1]) + m[a, 2] * p[:, 2]) + m[a, 3]) for a in range(3)], -1)


def pull(d, y):
    """x = D^-1(y) [n, 3] fp64 for network-frame points y [n, 3], and the pulled state (a [n, 4], det, u, v, h, k, inside)."""
    frame, h0, dh, kn = _table(d)
    eu, ev, eh, c = frame[0:3], frame[3:6], frame[6:9], frame[9:12]
    dd = [y[:, a] - c[a] for a in range(3)]

    def dot(e):
        return (e[0] * dd[0] + e[1] * dd[1]) + e[2] * dd[2]
    u, v, h = dot(eu), dot(ev), dot(eh)
    K = kn.shape[0]
    r = (h - h0) / dh
    kf = np.minimum(np.maximum(np.floor(r), 0.0), float(K - 2))
    k = kf.astype(np.int64)
    inside = (r >= 0.0) & (r <= float(K - 1))
    s = np.minimum(np.maximum(r - kf, 0.0), 1.0)
    k0, k1 = kn[k], kn[k + 1]
    e = k0 + s[:, None] * (k1 - k0)
    a, t = e[:, :4], e[:, 4:]
    det = a[:, 0] * a[:, 3] - a[:, 1] * a[:, 2]
    du, dv = u - t[:, 0], v - t[:, 1]
    up = (a[:, 3] * du - a[:, 1] * dv) / det
    vp = (a[:, 0] * dv - a[:, 2] * du) / det
    x = np.stack([((c[i] + up * eu[i]) + vp * ev[i]) + h * eh[i] for i in range(3)], -1)
    return x, dict(a=a, det=det, u=up, v=vp, h=h, k=k, inside=inside)


def forward(d, x):
    """D(x) [n, 3] fp64 (the map whose inverse pull is): (u, v) -> A(h) (u, v) + t(h), h kept."""
    frame, h0, dh, kn = _table(d)
    eu, ev, eh, c = frame[0:3], frame[3:6], frame[6:9], frame[9:12]
    dd = x - c[None, :]
    u, v, h = dd @ eu, dd @ ev, dd @ eh
    K = kn.shape[0]
    r = (h - h0) / dh
    kf = np.clip(np.floor(r), 0, K - 2)
    s = np.clip(r - kf, 0.0, 1.0)
    k = kf.astype(np.int64)
    e = kn[k] + s[:, None] * (kn[k + 1] - kn[k])
    uu = e[:, 0] * u + e[:, 1] * v + e[:, 4]
    vv = e[:, 2] * u + e[:, 3] * v + e[:, 5]
    return c[None, :] + uu[:, None] * eu[None, :] + vv[:, None] * ev[None, :] + h[:, None] * eh[None, :]


def targets(move, pts):
    """The fp32 targets [n, 3] of grid or sample points under a move: fp32(D^-1(trans p)) when deformed, E.targets otherwise."""
    trans = np.asarray(move["trans"], dtype=np.float64)[:3]
    if move.get("deform") is None:
        return E.targets(trans, pts)
    x, _ = pull(move["deform"], moved(trans, pts))
    return x.astype(np.float32)


def direction(d, st, w):
    """J_D^-1 w [n, 3] fp64 at the pulled state st (pull's) of directions w [n, 3] (network frame, fp64)."""
    frame, _, dh, kn = _table(d)
    eu, ev, eh = frame[0:3], frame[3:6], frame[6:9]

    def dot(e):
        return (e[0] * w[:, 0] + e[1] * w[:, 1]) + e[2] * w[:, 2]
    wu, wv, wh = dot(eu), dot(ev), dot(eh)
    k = st["k"]
    sl = (kn[k + 1] - kn[k]) / dh
    g0 = np.where(st["inside"], (sl[:, 0] * st["u"] + sl[:, 1] * st["v"]) + sl[:, 4], 0.0)
    g1 = np.where(st["inside"], (sl[:, 2] * st["u"] + sl[:, 3] * st["v"]) + sl[:, 5], 0.0)
    r0, r1 = wu - wh * g0, wv - wh * g1
    a, det = st["a"], st["det"]
    du = (a[:, 3] * r0 - a[:, 1] * r1) / det
    dv = (a[:, 0] * r1 - a[:, 2] * r0) / det
    return np.stack([(du * eu[i] + dv * ev[i]) + wh * eh[i] for i in range(3)], -1)


def target_dirs(move, pts, dirs):
    """The normalised fp32 view directions [n, 3] of a move's targets (render_moves_oracle.target_dirs when rigid)."""
    trans = np.asarray(move["trans"], dtype=np.float64)[:3]
    if move.get("deform") is None:
        return RM.target_dirs(trans, dirs)
    _, st = pull(move["deform"], moved(trans, pts))
    d = np.asarray(dirs, dtype=np.float32).astype(np.float64)
    w = np.stack([(trans[a, 0] * d[:, 0] + trans[a, 1] * d[:, 1]) + trans[a, 2] * d[:, 2] for a in range(3)], -1)
    dt = direction(move["deform"], st, w).astype(np.float32)
    nrm = np.sqrt((dt[:, 0] * dt[:, 0] + dt[:, 1] * dt[:, 1]) + dt[:, 2] * dt[:, 2])
    return (dt / nrm[:, None]).astype(np.float32)


def det_problem_interval(A, B):
    """Whether det(A + s (B - A)) <= 0 for some s in [0, 1], A and B 2x2: a quadratic in s, its minimum on [0, 1]."""
    A, B = np.asarray(A, dtype=np.float64).reshape(4), np.asarray(B, dtype=np.float64).reshape(4)
    D = B - A
    d0, a2 = A[0] * A[3] - A[1] * A[2], D[0] * D[3] - D[1] * D[2]
    b1 = ((A[0] * D[3] + D[0] * A[3]) - A[1] * D[2]) - D[1] * A[2]
    cand = [d0, (d0 + b1) + a2]
    if a2 > 0.0 and 0.0 < -b1 / (2.0 * a2) < 1.0:
        cand.append(d0 - (b1 * b1) / (4.0 * a2))
    return min(cand) <= 0.0


def destination_box(move, T, extents, dim, samples=0, rng=None):
    """The destination box of a deformed move's source box (collide.cu destination_box): the frame box of the source box's
    corners, the images of its horizontal corners at its two heights and at the knot heights between them, mapped by trans^-1
    to index space, floor / ceil, one voxel of margin, clipped -> (lo [3], hi [3])."""
    inv, b = E.grid_index_map(T, extents, dim)
    A = np.linalg.inv(inv)
    box = np.asarray(move["box"], dtype=np.float64)
    corners = np.array([[box[1] + 0.5 if c & 1 else box[0] - 0.5, box[3] + 0.5 if c & 2 else box[2] - 0.5,
                         box[5] + 0.5 if c & 4 else box[4] - 0.5] for c in range(8)])
    src = corners @ A.T + b[None, :]
    frame, h0, dh, kn = _table(move["deform"])
    F = frame[:9].reshape(3, 3)
    f = (src - frame[9:][None, :]) @ F.T
    lo, hi = f.min(0), f.max(0)
    hs = [lo[2], hi[2]] + [h0 + k * dh for k in range(kn.shape[0]) if lo[2] < h0 + k * dh < hi[2]]
    pts = []
    for h in hs:
        for c in range(4):
            fc = np.array([hi[0] if c & 1 else lo[0], hi[1] if c & 2 else lo[1], h])
            pts.append(frame[9:] + F.T @ fc)
    img = forward(move["deform"], np.array(pts))
    trans = np.asarray(move["trans"], dtype=np.float64)
    M = np.linalg.inv(trans[:3, :3])
    p = (img - trans[:3, 3][None, :]) @ M.T
    u = (p - b[None, :]) @ inv.T
    l, h = np.floor(u.min(0)) - 1, np.ceil(u.max(0)) + 1
    return np.clip(l, 0, dim).astype(np.int64), np.clip(h, -1, dim - 1).astype(np.int64)


# ---- the rules, with the target replaced -----------------------------------------------------------------------------------

def take_mask(o, pts, inv, b, move, evaluate, level):
    """group_oracle.take_mask with the deformed target -> (take, occ_t, label_t, evaluated)."""
    G = GO.group_of(move)
    lev = np.float32(level)
    t = targets(move, pts)
    idx = np.nonzero(E.in_box(E.index_of(inv, b, t), move["box"]))[0]
    take = np.zeros(o.shape[0], dtype=bool)
    occ_t = np.zeros(o.shape[0], dtype=np.float32)
    lab_t = np.zeros(o.shape[0], dtype=np.int64)
    if idx.size:
        o_t, l_t = evaluate(t[idx])
        l_t = np.asarray(l_t, dtype=np.int64)
        occ_t[idx], lab_t[idx] = o_t, l_t
        take[idx] = np.isin(l_t, G) & ((np.asarray(o_t) > lev) | (o[idx] <= lev)) & GO.keeps(move, t[idx], l_t)
    return take, occ_t, lab_t, int(idx.size)


def apply(o, lab, pts, inv, b, move, evaluate, level):
    if move.get("deform") is None:
        return GO.apply(o, lab, pts, inv, b, move, evaluate, level)
    take, occ_t, lab_t, n = take_mask(o, pts, inv, b, move, evaluate, level)
    vacate = GO.vacate_mask(o, lab, pts, move, level, take)
    o[take], lab[take] = occ_t[take], lab_t[take]
    o[vacate] = 0.0
    return n


def edit(occ, labels, T, extents, moves, evaluate, level):
    """The edited sweep with deformed moves -> (occ, labels, evaluated)."""
    dim = occ.shape[0]
    o, lab = occ.reshape(-1).astype(np.float32).copy(), labels.reshape(-1).astype(np.int64).copy()
    pts = E.sweep_points(T, extents, dim)
    inv, b = E.grid_index_map(T, extents, dim)
    n = sum(apply(o, lab, pts, inv, b, mv, evaluate, level) for mv in moves)
    return o.reshape(occ.shape), lab.reshape(occ.shape).astype(labels.dtype), n


def nearest_evaluate(occ, labels, inv, b):
    """evaluate() of the grid-only edit: the unedited grid at the target's nearest index (in the box, so in the grid)."""
    dim = occ.shape[0]
    o, lab = occ.reshape(-1), labels.reshape(-1)

    def f(t):
        q = np.rint(E.index_of(inv, b, t)).astype(np.int64)
        qi = (q[:, 0] * dim + q[:, 1]) * dim + q[:, 2]
        return o[qi], lab[qi]
    return f


def grid_edit(src_occ, src_labels, occ, labels, T, extents, moves, level):
    """group_oracle.grid_edit with deformed moves -> (occ, labels, landed [n], overwritten [n, 128])."""
    landed = np.zeros(len(moves), dtype=np.int64)
    overwritten = np.zeros((len(moves), N_LABELS), dtype=np.int64)
    state_o, state_l = occ.copy(), labels.copy()
    dim = occ.shape[0]
    pts = E.sweep_points(T, extents, dim)
    inv, b = E.grid_index_map(T, extents, dim)
    ev = nearest_evaluate(src_occ.astype(np.float32), src_labels.astype(np.int64), inv, b)
    lev = np.float32(level)
    for i, mv in enumerate(moves):
        if mv.get("deform") is None:
            state_o, state_l, land, over = GO.grid_edit(src_occ, src_labels, state_o, state_l, T, extents, [mv], level)
            landed[i], overwritten[i] = land[0], over[0]
            continue
        o, lab = state_o.reshape(-1).astype(np.float32).copy(), state_l.reshape(-1).astype(np.int64).copy()
        take, occ_t, lab_t, _ = take_mask(o, pts, inv, b, mv, ev, level)
        solid_take = take & (occ_t > lev)
        landed[i] = int(solid_take.sum())
        vacated = np.zeros_like(take) if mv.get("copy") else (np.isin(lab, GO.group_of(mv)) &
                                                              (GO.keeps(mv, pts, lab) | bool(mv.get("rest_drop", False))))
        overwritten[i] = np.bincount(lab[solid_take & (o > lev) & ~vacated], minlength=N_LABELS)
        vacate = GO.vacate_mask(o, lab, pts, mv, level, take)
        o[take], lab[take] = occ_t[take], lab_t[take]
        o[vacate] = 0.0
        state_o, state_l = o.reshape(occ.shape), lab.reshape(occ.shape).astype(labels.dtype)
    return state_o, state_l, landed, overwritten


def moved_object(occ, labels, T, extents, move, level):
    """group_oracle.moved_object with the deformed target: bool [dim]^3."""
    dim = occ.shape[0]
    o, lab = occ.reshape(-1).astype(np.float32), labels.reshape(-1).astype(np.int64)
    pts = E.sweep_points(T, extents, dim)
    inv, b = E.grid_index_map(T, extents, dim)
    t = targets(move, pts)
    u = E.index_of(inv, b, t)
    src = E.in_box(u, move["box"])
    q = np.rint(u[src]).astype(np.int64)
    qi = (q[:, 0] * dim + q[:, 1]) * dim + q[:, 2]
    ok = np.isin(lab[qi], GO.group_of(move)) & (o[qi] > np.float32(level)) & GO.keeps(move, t[src], lab[qi])
    src[np.nonzero(src)[0]] = ok
    return src.reshape(occ.shape)


def move_overlap(occ, labels, T, extents, moves, level, obstacles=None):
    """group_oracle.move_overlap with deformed moves, over the whole grid -> (overlap [n, 128], landed [n])."""
    overlap = np.zeros((len(moves), N_LABELS), dtype=np.int64)
    landed = np.zeros(len(moves), dtype=np.int64)
    lab = labels.reshape(-1).astype(np.int64)
    is_obst = np.ones(N_LABELS, dtype=bool) if obstacles is None else np.isin(np.arange(N_LABELS), list(obstacles))
    blocking = (occ.reshape(-1) > np.float32(level)) & is_obst[np.clip(lab, 0, N_LABELS - 1)]
    for i, mv in enumerate(moves):
        if mv.get("deform") is None:
            over, land = GO.move_overlap(occ, labels, T, extents, [mv], level, obstacles)
            overlap[i], landed[i] = over[0], land[0]
            continue
        S = moved_object(occ, labels, T, extents, mv, level).reshape(-1)
        landed[i] = int(S.sum())
        overlap[i] = np.bincount(lab[S & blocking & ~GO.vacated(occ, labels, T, extents, mv, level).reshape(-1)],
                                 minlength=N_LABELS)
    return overlap, landed


def render_apply_moves(raw, rays_o, rays_d, z, moves, T, extents, dim, evaluate, level, voxel, record=None):
    """group_oracle.render_apply_moves with deformed targets and view directions -> (edited copy, evaluated)."""
    out = raw.clone()
    n, s, c = out.shape
    flat = out.reshape(n * s, c)
    pts = RM.RO.sample_points(RM._np(rays_o), RM._np(rays_d), RM._np(z)).reshape(-1, 3)
    dirs = np.repeat(RM._np(rays_d), s, axis=0)
    inv, b = E.grid_index_map(T, extents, dim)
    lev = np.float32(level)
    ev = 0
    for mv in moves:
        if mv.get("deform") is None:
            o2, e2 = GO.render_apply_moves(flat.reshape(n, s, c), rays_o, rays_d, z, [mv], T, extents, dim, evaluate, level, voxel,
                                           record)
            flat.copy_(o2.reshape(n * s, c))
            ev += e2
            continue
        G = GO.group_of(mv)
        t = targets(mv, pts)
        inb = E.in_box(E.index_of(inv, b, t), mv["box"])
        pin = E.in_box(E.index_of(inv, b, pts), mv["box"])
        dev = flat.device
        o_p = RM.occupancy(flat[:, 3], voxel).cpu().numpy()
        l_p = RM.object_labels(flat).cpu().numpy()
        idx = np.nonzero(inb)[0]
        take = np.zeros(flat.shape[0], dtype=bool)
        rows = None
        if idx.size:
            rows = evaluate(t[idx], target_dirs(mv, pts[idx], dirs[idx])).to(dev)
            lt = RM.object_labels(rows).cpu().numpy()
            ot = RM.occupancy(rows[:, 3], voxel).cpu().numpy()
            take[idx] = np.isin(lt, G) & ((ot > lev) | (o_p[idx] <= lev)) & GO.keeps(mv, t[idx], lt)
        vacate = np.zeros(flat.shape[0], dtype=bool)
        if not mv.get("copy"):
            keeps_p = GO.keeps(mv, pts, l_p)
            vacate = ~take & np.isin(l_p, G) & ((keeps_p & pin) | (bool(mv.get("rest_drop", False)) & ~keeps_p))
        if idx.size:
            took = take[idx]
            flat[torch.as_tensor(idx[took], device=dev)] = rows[torch.as_tensor(took, device=dev)]
        flat[torch.as_tensor(np.nonzero(vacate)[0], device=dev), 3] = 0.0
        if record is not None:
            record.append((take, vacate))
        ev += int(idx.size)
    return out, ev


def render_on_depths(rays_o, rays_d, p_coarse, p_fine, z_coarse, z_fine, moves, T, extents, dim, level, voxel, record=None):
    """group_oracle.render_on_depths with deformed moves: both passes teacher-forced on given depths."""
    dtype = next(iter(p_coarse.values())).dtype
    o, d = rays_o.float(), rays_d.float()
    vd = (d.double() / torch.norm(d.double(), dim=-1, keepdim=True)).to(dtype)
    out = {}
    for tag, p, z in (("coarse", p_coarse, z_coarse), ("fine", p_fine, z_fine)):
        z = z.float()
        pts = o[:, None, :] + d[:, None, :] * z[..., None]
        x = torch.cat([RM.embed(pts.reshape(-1, 3).to(dtype), 10), RM.embed(vd[:, None].expand(pts.shape).reshape(-1, 3), 4)], -1)
        raw = RM.mlp_forward(p, x).reshape(z.shape[0], z.shape[1], -1)
        rec = None if record is None else record.setdefault(tag, [])
        raw, ev = render_apply_moves(raw, o, d, z, moves, T, extents, dim, RM.network_evaluate(p, dtype), level, voxel, rec)
        rgb, w, depth, ins, acc = RM.composite(raw, z.to(dtype), d.to(dtype))
        out.update({"rgb_" + tag: rgb, "weights_" + tag: w, "depth_" + tag: depth, "ins_" + tag: ins, "acc_" + tag: acc,
                    "raw_" + tag: raw, "evaluated_" + tag: ev})
    return out
