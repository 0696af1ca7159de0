"""Multi-GPU plumbing for the render path (SURVEY.md 8e): rays are independent units, so a frame (or a
trajectory) is split into contiguous ray ranges per rank with the weights replicated, each rank renders its
slab with the fused kernels, and ONE all-gather of the packed image slabs assembles the result on every rank.
No collective sits on the data path of the kernels themselves.  world_of / all_gather / all_reduce_sum_ are the collectives
of the training losses and of data-parallel training: one process (no process group) is world 1, where they do nothing."""
import torch


def shard_range(n_items, world, rank, multiple=1):
    """Contiguous [lo, hi) of `n_items` for `rank`; every shard but the last is a multiple of `multiple` and all
    shards have equal padded length (returned as third value) so a fixed-size all-gather can be used."""
    per = -(-n_items // world)
    per = -(-per // multiple) * multiple
    lo = min(rank * per, n_items)
    hi = min(lo + per, n_items)
    return lo, hi, per


def world_of(group=None):
    """(world size, rank) of `group`; (1, 0) when torch.distributed is not initialised (one process)."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()):
        return 1, 0
    return dist.get_world_size(group), dist.get_rank(group)


def _nccl(group):
    import torch.distributed as dist
    return dist.get_backend(group) == "nccl"


def all_gather(t, group=None):
    """[W, *t.shape] on t's device, rank order.  NCCL gathers device tensors; gloo has no CUDA all-gather, so a gloo group is
    staged through host memory."""
    world, _ = world_of(group)
    if world == 1:
        return t[None]
    import torch.distributed as dist
    t = t.contiguous()
    if _nccl(group):
        out = t.new_empty((world,) + tuple(t.shape))
        dist.all_gather_into_tensor(out, t, group=group)
        return out
    host = t.cpu()
    parts = [torch.empty_like(host) for _ in range(world)]
    dist.all_gather(parts, host, group=group)
    return torch.stack(parts).to(t.device)


def all_reduce_sum_(t, group=None):
    """In-place sum of `t` over the ranks (staged through host memory for gloo)."""
    world, _ = world_of(group)
    if world == 1:
        return t
    import torch.distributed as dist
    if _nccl(group):
        dist.all_reduce(t, group=group)
    else:
        host = t.cpu()
        dist.all_reduce(host, group=group)
        t.copy_(host)
    return t


IMAGE_KEYS = ("rgb_fine", "depth_fine", "acc_fine", "ins_fine")


def pack_image(out, keys=IMAGE_KEYS):
    """[n, 3 + 1 + 1 + ins] packed slab of the per-ray outputs that make up the rendered image."""
    cols = [out[k] if out[k].dim() == 2 else out[k][:, None] for k in keys]
    return torch.cat(cols, -1).contiguous()


def unpack_image(packed, ins_num, keys=IMAGE_KEYS):
    widths = {"rgb_fine": 3, "depth_fine": 1, "acc_fine": 1, "ins_fine": ins_num}
    res, c = {}, 0
    for k in keys:
        w = widths[k]
        res[k] = packed[..., c:c + w] if w > 1 or k == "ins_fine" else packed[..., c]
        c += w
    return res


def gather_image(out, world, group=None, pad_to=None):
    """All-gather the packed image slab of every rank: returns [world, n_pad, 5 + ins] on every rank."""
    import torch.distributed as dist
    slab = pack_image(out)
    if pad_to is not None and slab.shape[0] < pad_to:
        slab = torch.cat([slab, slab.new_zeros(pad_to - slab.shape[0], slab.shape[1])], 0)
    full = slab.new_empty((world * slab.shape[0],) + tuple(slab.shape[1:]))
    dist.all_gather_into_tensor(full, slab, group=group)
    return full.view((world,) + tuple(slab.shape))


def render_frame_sharded(rays_o, rays_d, model_coarse, model_fine, z_vals_coarse, N_importance=128, render_fn=None,
                         group=None):
    """Render one frame split across the ranks of the default process group (strong scaling over rays) and return
    the full-frame image dict on every rank.  `render_fn` defaults to the CUDA renderer."""
    import torch.distributed as dist
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    if render_fn is None:
        from .render import render_rays as render_fn
    n = rays_o.shape[0]
    lo, hi, per = shard_range(n, world, rank, multiple=128)
    out = render_fn(rays_o[lo:hi], rays_d[lo:hi], model_coarse, model_fine, z_vals_coarse, N_importance=N_importance,
                    want_raw=False, want_coarse=False)
    ins_num = out["ins_fine"].shape[-1]
    full = gather_image(out, world, group=group, pad_to=per)                 # [world, per, 5+ins]
    flat = full.reshape(world * per, -1)[:n]
    return unpack_image(flat, ins_num)


def render_camera_sharded(H, W, K, c2w, near, far, model_coarse, model_fine, N_samples=64, N_importance=128, frame_fn=None,
                          group=None, device=None):
    """One camera of a trajectory (BASELINE config 5; the per-pose loop of render_test, tester.py:55-76) split by pixel range
    across the ranks: every rank runs the frame driver (rays generated on its own device from K / c2w) on its range and ONE
    all-gather assembles the image dict {"rgb" [H,W,3], "ins" [H,W,ins_num], "depth" [H,W], "acc" [H,W]} on every rank.
    `frame_fn(H, W, K, c2w, near, far, mc, mf, N_samples=, N_importance=, pixel_range=)` defaults to render.render_frame."""
    import torch.distributed as dist
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    if frame_fn is None:
        from .render import render_frame as frame_fn
    n = H * W
    lo, hi, per = shard_range(n, world, rank, multiple=128)
    part = frame_fn(H, W, K, c2w, near, far, model_coarse, model_fine, N_samples=N_samples, N_importance=N_importance,
                    pixel_range=(lo, hi - lo))
    out = {"rgb_fine": part["rgb"], "depth_fine": part["depth"], "acc_fine": part["acc"], "ins_fine": part["ins"]}
    if device is not None:                                  # NCCL gathers device tensors; the frame driver returns host maps
        out = {k: v.to(device, non_blocking=True) for k, v in out.items()}
    ins_num = out["ins_fine"].shape[-1]
    full = gather_image(out, world, group=group, pad_to=per)
    img = unpack_image(full.reshape(world * per, -1)[:n], ins_num)
    return {"rgb": img["rgb_fine"].reshape(H, W, 3), "ins": img["ins_fine"].reshape(H, W, ins_num),
            "depth": img["depth_fine"].reshape(H, W), "acc": img["acc_fine"].reshape(H, W)}


def render_trajectory_sharded(poses, H, W, K, near, far, model_coarse, model_fine, **kw):
    """Generator over a camera trajectory (e.g. the 900 poses of Replica office_2): yields the assembled image dict per pose."""
    for c2w in poses:
        yield render_camera_sharded(H, W, K, c2w, near, far, model_coarse, model_fine, **kw)
