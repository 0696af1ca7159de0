"""CPU oracle of rendering moved objects per sample -- TEST INFRASTRUCTURE ONLY (the product package never imports it).

Restates DESIGN.md, "Rendering moved objects", one rounding per operation, on top of edit_sweep_oracle's target and index
computation, dmnerf_oracle's network and composite and region_oracle's piece test.  Per move and sample p = o + d z (fp32) with raw
row r_p (torch, any device), o_p = 1 - exp(-relu(r_p[3]) voxel) and label_p = argmax(sigmoid(r_p[4:])), first maximum:
  target     t = fp32(trans p) and its nearest index, as edit_sweep_oracle computes them; the view direction
             fp32(trans[:3, :3] d) (fp64, left to right), normalised by sqrt((x^2 + y^2) + z^2) and divided in fp32;
  take       t's index in the box && label(t) == mv && (occ(t) > level || o_p <= level) && (no piece || the piece keeps t):
             r_p = the network's row at (t, its direction);
  vacate     otherwise label_p == mv && ((the piece keeps p, every p without one) && p's index in the box
                                         || rest_drop && the piece does not keep p): r_p[3] = 0.
The network at the targets is a callback evaluate(t [m, 3], dirs [m, 3]) -> rows [m, C]: the device network for bit-level
checks, or network_evaluate's fp64 oracle network."""
import numpy as np
import torch

from oracle import edit_sweep_oracle as ES
from oracle import region_oracle as RO
from oracle.dmnerf_oracle import composite, embed, mlp_forward
from oracle.objects_oracle import object_labels


def target_dirs(trans, dirs):
    """The targets' view directions [n, 3] float32: fp32(trans[:3, :3] d) in fp64, normalised in fp32 as the prologue does."""
    m = np.asarray(trans, dtype=np.float64)
    d = np.asarray(dirs, dtype=np.float32).astype(np.float64)
    r = np.stack([(m[a, 0] * d[:, 0] + m[a, 1] * d[:, 1]) + m[a, 2] * d[:, 2] for a in range(3)], -1).astype(np.float32)
    nrm = np.sqrt((r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1]) + r[:, 2] * r[:, 2])
    return (r / nrm[:, None]).astype(np.float32)


def occupancy(a, voxel):
    """occ = 1 - exp(-relu(a) voxel), fp32 torch ops on a's device."""
    return 1.0 - torch.exp(-torch.relu(a) * torch.tensor(np.float32(voxel), device=a.device))


def apply_move(raw, pts, dirs, move, inv, b, evaluate, level, voxel, record=None):
    """One move on the rows raw [n, C] (torch, edited in place) of the samples pts [n, 3] with ray directions dirs [n, 3] (numpy
    fp32) -> the number of targets evaluated.  move: dict(label, trans (4x4 or 3x4), box, piece (edit_sweep_oracle.Piece or
    None), rest_drop).  record (a list, or None): receives the move's decisions (take [n], vacate [n], bool numpy)."""
    mv, piece = int(move["label"]), move.get("piece")
    lev = np.float32(level)
    trans = np.asarray(move["trans"], dtype=np.float64)[:3]
    t = ES.targets(trans, pts)
    inb = ES.in_box(ES.index_of(inv, b, t), move["box"])
    pin = ES.in_box(ES.index_of(inv, b, pts), move["box"])
    dev = raw.device
    o_p = occupancy(raw[:, 3], voxel).cpu().numpy()
    l_p = object_labels(raw).cpu().numpy()
    idx = np.nonzero(inb)[0]
    take = np.zeros(raw.shape[0], dtype=bool)
    rows = None
    if idx.size:
        rows = evaluate(t[idx], target_dirs(trans, dirs[idx])).to(dev)
        lt = object_labels(rows).cpu().numpy()
        ot = occupancy(rows[:, 3], voxel).cpu().numpy()
        ok = (lt == mv) & ((ot > lev) | (o_p[idx] <= lev))
        if piece is not None:
            ok &= piece.keeps(t[idx])
        take[idx] = ok
    keeps_p = np.ones(raw.shape[0], dtype=bool) if piece is None else piece.keeps(pts)
    vacate = ~take & (l_p == mv) & ((keeps_p & pin) | (bool(move.get("rest_drop", False)) & ~keeps_p))
    if idx.size:
        took = take[idx]
        raw[torch.as_tensor(idx[took], device=dev)] = rows[torch.as_tensor(took, device=dev)]
    raw[torch.as_tensor(np.nonzero(vacate)[0], device=dev), 3] = 0.0
    if record is not None:
        record.append((take, vacate))
    return int(idx.size)


def apply_moves(raw, rays_o, rays_d, z, moves, T, extents, dim, evaluate, level, voxel, record=None):
    """The moves applied in order to the rows raw [N, S, C] (torch) of samples o + d z (z [N, S]) -> (edited copy, evaluated).
    record: as apply_move, one entry per move, over the N * S samples."""
    out = raw.clone()
    n, s, c = out.shape
    flat = out.reshape(n * s, c)
    pts = RO.sample_points(_np(rays_o), _np(rays_d), _np(z)).reshape(-1, 3)
    dirs = np.repeat(_np(rays_d), s, axis=0)
    inv, b = ES.grid_index_map(T, extents, dim)
    ev = 0
    for mv in moves:
        ev += apply_move(flat, pts, dirs, mv, inv, b, evaluate, level, voxel, record)
    return out, ev


def _np(x):
    return x.detach().cpu().float().numpy() if torch.is_tensor(x) else np.asarray(x, dtype=np.float32)


def network_evaluate(p, dtype=torch.float64):
    """evaluate() of the oracle network p (a state dict of tensors): points mode, the directions embedded as given."""
    dev = next(iter(p.values())).device

    def f(t, dirs):
        x = torch.cat([embed(torch.as_tensor(t, dtype=dtype, device=dev), 10), embed(torch.as_tensor(dirs, dtype=dtype, device=dev), 4)],
                      -1)
        return mlp_forward(p, x)
    return f


def render_on_depths(rays_o, rays_d, p_coarse, p_fine, z_coarse, z_fine, moves, T, extents, dim, level, voxel, record=None):
    """Both passes on given depths (teacher-forced: a kernel's own z_vals): the network p (state dicts, their dtype, fp64 for
    the reference) on the fp32 sample points o + d z and the fp32 unit view directions, the moves applied (decisions taken on the
    fp32 points, the targets through network_evaluate), then dmnerf_oracle's composite in that dtype.  record: {"coarse": [...],
    "fine": [...]} of apply_moves' decisions, or None.  Returns both passes' maps and edited rows."""
    dtype = next(iter(p_coarse.values())).dtype
    o, d = rays_o.float(), rays_d.float()
    vd = (d.double() / torch.norm(d.double(), dim=-1, keepdim=True)).to(dtype)
    out = {}
    for tag, p, z in (("coarse", p_coarse, z_coarse), ("fine", p_fine, z_fine)):
        z = z.float()
        pts = o[:, None, :] + d[:, None, :] * z[..., None]                     # the prologue's fp32 point
        x = torch.cat([embed(pts.reshape(-1, 3).to(dtype), 10), embed(vd[:, None].expand(pts.shape).reshape(-1, 3), 4)], -1)
        raw = mlp_forward(p, x).reshape(z.shape[0], z.shape[1], -1)
        rec = None if record is None else record.setdefault(tag, [])
        raw, ev = apply_moves(raw, o, d, z, moves, T, extents, dim, network_evaluate(p, dtype), level, voxel, rec)
        rgb, w, depth, ins, acc = composite(raw, z.to(dtype), d.to(dtype))
        out.update({"rgb_" + tag: rgb, "weights_" + tag: w, "depth_" + tag: depth, "ins_" + tag: ins, "acc_" + tag: acc,
                    "raw_" + tag: raw, "evaluated_" + tag: ev})
    return out
