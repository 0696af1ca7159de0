"""networks/penalizer.py on the native kernels (csrc/penalizer.cu): the "emptiness" regulariser on the per-sample object
logits, forward and backward, with the reference's signatures.

    emptiness_penalizer(raw, z_vals, depths, rays_d, tolerance, deta_w)      reference networks/penalizer.py:5-55
    ins_penalizer(raw, z_vals, depth, rays_d, args)                          reference networks/penalizer.py:58-62

Both return a tensor of shape [1] like the reference (its `torch.maximum(..., torch.tensor([1e-8]))` broadcasts the scalar).
Gradient flows to `raw[..., 4:]` only: the depth is detached by the reference and z_vals / rays_d carry no gradient there.
The forward sums in an order fixed by the sizes, so the loss and its gradient are reproducible bit for bit.  The same Function
serves a batch split over the ranks of a process group (distributed.ins_penalizer_sharded), of which one process is the
one-shard case.
"""
import torch

from . import _lib
from .engine import get_context
from .parallel import all_gather, world_of


class _Penalizer(torch.autograd.Function):
    """forward(raw, z_vals, depth, rays_d, tolerance, deta_w, group): the loss of the rows given.  Over the W ranks of `group`
    each rank's mask populations and masked sums (the head of its partials buffer) are gathered and merged in rank order, so
    every rank gets the loss of the whole batch and the state its backward reads."""

    @staticmethod
    def forward(fctx, raw, z_vals, depth, rays_d, tolerance, deta_w, group):
        if not raw.is_cuda:
            raise RuntimeError("emptiness_penalizer: expected CUDA tensors (no CPU fallback)")
        ctx = get_context(raw.device)
        raw_c = raw.detach().contiguous().float()
        z_c = z_vals.detach().contiguous().float()
        d_c = depth.detach().reshape(-1).contiguous().float()
        rd_c = rays_d.detach().contiguous().float()
        n, s, c = raw_c.shape
        if z_c.shape != (n, s) or d_c.shape != (n,) or rd_c.shape != (n, 3):
            raise RuntimeError("emptiness_penalizer: inconsistent shapes raw %s z_vals %s depth %s rays_d %s"
                               % (tuple(raw.shape), tuple(z_vals.shape), tuple(depth.shape), tuple(rays_d.shape)))
        u8 = torch.uint8
        part = torch.empty(int(ctx.lib.dmnerf_penalizer_partials_bytes(n, s, c)), device=raw.device, dtype=u8)
        loss = torch.empty(1, device=raw.device, dtype=torch.float32)
        ctx.call("dmnerf_penalizer_forward", _lib.ptr(raw_c), _lib.ptr(z_c), _lib.ptr(d_c), _lib.ptr(rd_c), n, s, c, float(tolerance),
                 float(deta_w), _lib.ptr(part, u8), _lib.ptr(loss))
        state = part[:int(ctx.lib.dmnerf_penalizer_state_bytes())]
        world, _ = world_of(group)
        if world > 1:
            heads = all_gather(state, group)
            state = torch.empty_like(state)
            ctx.call("dmnerf_penalizer_merge", _lib.ptr(heads, u8), world, c, _lib.ptr(state, u8), _lib.ptr(loss))
        fctx.save_for_backward(raw_c, z_c, d_c, rd_c, state)
        fctx.cfg = (float(tolerance), float(deta_w))
        return loss

    @staticmethod
    def backward(fctx, g_loss):
        raw_c, z_c, d_c, rd_c, state = fctx.saved_tensors
        ctx = get_context(raw_c.device)
        n, s, c = raw_c.shape
        d_raw = torch.empty_like(raw_c)           # the kernel writes every channel (zeros for rgb / sigma)
        g = g_loss.detach().reshape(-1)[:1].contiguous().float()
        ctx.call("dmnerf_penalizer_backward", _lib.ptr(raw_c), _lib.ptr(z_c), _lib.ptr(d_c), _lib.ptr(rd_c), n, s, c, fctx.cfg[0],
                 fctx.cfg[1], _lib.ptr(state, torch.uint8), _lib.ptr(g), _lib.ptr(d_raw), 0)
        return d_raw, None, None, None, None, None, None


def emptiness_penalizer(raw, z_vals, depths, rays_d, tolerance, deta_w):
    """reference networks/penalizer.py:5-55; depths [N,1] (or [N]) is used as a constant."""
    return _Penalizer.apply(raw, z_vals, depths, rays_d, tolerance, deta_w, None)


def ins_penalizer(raw, z_vals, depth, rays_d, args):
    """reference networks/penalizer.py:58-62: reads args.tolerance and args.deta_w."""
    return emptiness_penalizer(raw, z_vals, depth[..., None].detach(), rays_d, args.tolerance, args.deta_w)
