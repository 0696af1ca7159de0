"""Drop-in for reference networks/render.py: `dm_nerf` (:31-96, the north_star's render_rays) and
`render_train` (:6-28, raw2outputs), running on the fused native kernels through the C ABI."""
import ctypes as C

import torch

from . import _lib
from .engine import get_context

KEYS = ("rgb_fine", "ins_fine", "z_vals_fine", "raw_fine", "raw_coarse", "rgb_coarse", "ins_coarse",
        "z_vals_coarse", "depth_fine", "depth_coarse")


def render_train(raw, z_vals, rays_d, keep_all_ins=False):
    """sigma->alpha exclusive-scan composite (render.py:6-28).  Returns (rgb_map, weights, depth_map, ins_map)."""
    from .autograd import _needs_grad
    if _needs_grad(raw):
        from .backward import CompositeFunction
        return CompositeFunction.apply(raw, z_vals, rays_d, keep_all_ins)
    rgb, w, depth, ins, _acc = composite(raw, z_vals, rays_d, keep_all_ins)
    return rgb, w, depth, ins


def composite(raw, z_vals, rays_d, keep_all_ins=False, keep_objects=None):
    """Inference composite -> (rgb, weights, depth, ins, acc).  keep_objects: object selection (labels in [0, C - 5]) as in
    render_rays: samples labelled otherwise enter with alpha = 0."""
    if not raw.is_cuda:
        raise RuntimeError("render_train: expected CUDA tensors (no CPU fallback)")
    n, s, c = raw.shape
    raw, z_vals, rays_d = raw.contiguous().float(), z_vals.contiguous().float(), rays_d.contiguous().float()
    dev = raw.device
    n_ins = c - 4 if keep_all_ins else c - 5
    rgb = torch.empty((n, 3), device=dev); w = torch.empty((n, s), device=dev)
    depth = torch.empty((n,), device=dev); acc = torch.empty((n,), device=dev)
    ins = torch.empty((n, n_ins), device=dev)
    from .objects import object_mask
    keep = None if keep_objects is None else _lib.keep_mask(object_mask(c - 5, keep=keep_objects))
    get_context(dev).call("dmnerf_composite", _lib.ptr(raw), _lib.ptr(z_vals), _lib.ptr(rays_d), n, s, c, int(keep_all_ins), keep,
                          _lib.ptr(rgb), _lib.ptr(w), _lib.ptr(depth), _lib.ptr(ins), _lib.ptr(acc))
    return rgb, w, depth, ins, acc


def bind_pair(ctx, model_coarse, model_fine):
    """Bind the coarse network to slot 0 and the fine one to slot 1 -> their common ins_num."""
    ins_num = ctx.bind(0, model_coarse)
    if ctx.bind(1, model_fine) != ins_num:
        raise RuntimeError("coarse and fine networks disagree on ins_num")
    return ins_num


def coarse_depths(z_vals_coarse, n):
    """z_vals_coarse of n rays -> (z_in, z_row_stride) of the C ABI: one shared row (a [S] tensor or the stride-0 expand of
    z_val_sample) with stride 0, or one row per ray with stride S."""
    if z_vals_coarse.dim() == 1:
        return z_vals_coarse.contiguous().float(), 0
    if z_vals_coarse.dim() == 2 and z_vals_coarse.shape[0] > 1 and z_vals_coarse.stride(0) == 0:
        return z_vals_coarse[0].contiguous().float(), 0
    z_in = z_vals_coarse.contiguous().float()
    if z_in.shape[0] != n:
        raise RuntimeError("z_vals_coarse has %d rows for %d rays" % (z_in.shape[0], n))
    return z_in, z_vals_coarse.shape[-1]


def reference_draws(perturb, n, S, N_importance, device, t_rand=None, u=None):
    """The uniforms of a perturbed render, drawn where the caller did not pass them, in the reference's order: t_rand [n, S]
    (render.py:46), then u [n, N_importance] (helpers.py:135).  (None, None) when perturb <= 0."""
    if perturb <= 0.0:
        return None, None
    if t_rand is None:
        t_rand = torch.rand((n, S), device=device)
    if u is None:
        u = torch.rand((n, N_importance), device=device)
    return t_rand.contiguous().float(), u.contiguous().float()


def scene_edit(who, ins_num, device, model_coarse, model_fine, keep_objects=None, region=None, appearance=None):
    """The scene edit of an inference entry point rendering on `device` with networks of ins_num: keep_objects (labels in
    [0, ins_num]), region (objects.Region) and appearance (objects.Appearance) -> (a pointer to the _lib.Edit for io.edit, or
    None without an edit; the ctypes objects it points into, which the caller holds until the native call returns).  The
    edits render inference only: RuntimeError when the networks would record gradients.  ValueError for a region whose bits
    live on another device or an appearance built for another ins_num."""
    if keep_objects is None and region is None and appearance is None:
        return None, ()
    from .autograd import _needs_grad
    if _needs_grad(model_coarse, model_fine):
        raise RuntimeError("%s: a scene edit (object selection, region, appearance) is inference-only; call it under "
                           "torch.no_grad() or with parameters that do not require grad" % who)
    edit, held = _lib.Edit(), []
    if keep_objects is not None:
        from .objects import object_mask
        keep = _lib.keep_mask(object_mask(ins_num, keep=keep_objects))
        edit.keep = C.cast(keep, C.POINTER(C.c_uint32))
        held.append(keep)
    if region is not None:
        if region.bits.device != torch.device(device):
            raise ValueError("region: bits live on %s, the render on %s" % (region.bits.device, device))
        desc = region.abi(ins_num)
        edit.region = C.pointer(desc)
        held += [desc, region.bits]
    if appearance is not None:
        if appearance.ins_num != ins_num:
            raise ValueError("appearance: built for ins_num %d, the networks have ins_num %d" % (appearance.ins_num, ins_num))
        table = _lib.floats(appearance.table, appearance.table.size)
        edit.appearance, edit.appearance_labels = C.cast(table, C.POINTER(C.c_float)), ins_num + 1
        held.append(table)
    return C.pointer(edit), held


def _check_embedders(position_embedder, view_embedder):
    pd = getattr(position_embedder, "out_dim", None)
    vd = getattr(view_embedder, "out_dim", None)
    if pd != 63 or vd != 27:
        raise NotImplementedError("the fused renderer is specialised for get_embedder(10) / get_embedder(4) "
                                  "(63 + 27 channels, config.py:128-129); got out_dim %s / %s" % (pd, vd))


def render_rays(rays_o, rays_d, model_coarse, model_fine, z_vals_coarse, perturb=0.0, N_importance=128,
                t_rand=None, u=None, want_raw=True, want_coarse=True, want_samples=None, keep_all_ins=False,
                impl=_lib.IMPL_AUTO, keep_objects=None, region=None, appearance=None, moves=None):
    """Whole per-ray pipeline on the device.  Returns the reference's dict keys plus acc / weights maps.
    want_raw: per-sample network outputs raw_* (forces the stage-by-stage kernels); want_samples: per-sample depths and
    weights (z_vals_*, weights_*; default = want_raw); want_coarse: the coarse pass' maps.  With want_raw=False and
    64 + 128 samples the whole call is ONE kernel and only the requested per-ray maps are written.
    keep_objects: an iterable of object labels in [0, ins_num]; samples labelled otherwise get alpha = 0 in both passes
    (DESIGN.md, "Object selection").  raw_* stay the network's output.  Inference only.
    region: an objects.Region; samples it drops get alpha = 0 in both passes as well (DESIGN.md, "Region selection").
    appearance: an objects.Appearance; every sample the selection and the region keep has its label's density scale and colour
    map applied in both passes (DESIGN.md, "Object appearance").  Inference only.
    impl: _lib.IMPL_UMMA_F16 runs the fp16 preview network (DESIGN.md section 10); IMPL_AUTO follows DMNERF_INFER_IMPL.
    moves: an objects.MovedScene (objects.render_moves): the moves applied per sample to each pass's network output before its
    composite, by the edited sweep's rule (DESIGN.md, "Rendering moved objects"), always on the stage kernels; raw_* are the edited
    rows and the result gains evaluated = (coarse, fine) targets.  Composes with keep_objects, region and appearance.  Inference
    only; not with _lib.IMPL_SIMT."""
    impl = _lib.infer_impl(impl)
    if want_samples is None:
        want_samples = want_raw
    dev = rays_o.device
    if dev.type != "cuda":
        raise RuntimeError("dm_nerf: expected CUDA tensors (no CPU fallback)")
    ctx = get_context(dev)
    ins_num = bind_pair(ctx, model_coarse, model_fine)
    edit, held = scene_edit("render_rays", ins_num, dev, model_coarse, model_fine, keep_objects, region, appearance)
    if moves is not None:
        _check_moved(moves, "render_rays", dev, model_coarse, model_fine)
    rays_o = rays_o.reshape(-1, 3).contiguous().float()
    rays_d = rays_d.reshape(-1, 3).contiguous().float()
    n = rays_o.shape[0]
    S = z_vals_coarse.shape[-1]
    F, ch = S + N_importance, 4 + ins_num + 1
    z_in, z_stride = coarse_depths(z_vals_coarse, n)
    t_rand, u = reference_draws(perturb, n, S, N_importance, dev, t_rand, u)
    flags = _lib.FLAG_PERTURB if perturb > 0.0 else 0
    if want_raw:
        flags |= _lib.FLAG_WANT_RAW
    if keep_all_ins:
        flags |= _lib.FLAG_KEEP_INS
    n_ins_out = ins_num + 1 if keep_all_ins else ins_num
    e = lambda *shape: torch.empty(shape, device=dev, dtype=torch.float32)
    out = {"rgb_fine": e(n, 3), "ins_fine": e(n, n_ins_out), "depth_fine": e(n), "acc_fine": e(n)}
    if want_samples or want_raw:
        out.update({"z_vals_fine": e(n, F), "weights_fine": e(n, F), "z_vals_coarse": e(n, S)})
    if want_coarse:
        out.update({"rgb_coarse": e(n, 3), "ins_coarse": e(n, n_ins_out), "depth_coarse": e(n), "acc_coarse": e(n)})
        if want_samples or want_raw:
            out["weights_coarse"] = e(n, S)
    if want_raw:
        out.update({"raw_fine": e(n, F, ch), "raw_coarse": e(n, S, ch)})
    io = _lib.RenderIO()
    io.rays_o, io.rays_d, io.z_coarse, io.z_row_stride = _lib.ptr(rays_o), _lib.ptr(rays_d), _lib.ptr(z_in), z_stride
    io.t_rand, io.u = _lib.ptr(t_rand), _lib.ptr(u)
    for k, v in out.items():
        setattr(io, k, _lib.ptr(v))
    io.edit = edit
    if moves is None:
        ctx.call("dmnerf_render_forward", ctx.handle, io, n, S, N_importance, flags, impl)
        return out
    evaluated = (C.c_int64 * 2)()
    if moves.deformation_array() is not None:
        ctx.call("dmnerf_render_moved_deformed", ctx.handle, io, n, S, N_importance, flags, impl, C.byref(moves.abi()),
                 moves.copy_flags(), moves.group_words(), moves.deformation_array(), evaluated)
    elif moves.group_words() is not None:
        ctx.call("dmnerf_render_moved_groups", ctx.handle, io, n, S, N_importance, flags, impl, C.byref(moves.abi()),
                 moves.copy_flags(), moves.group_words(), evaluated)
    elif moves.copy_flags() is None:
        ctx.call("dmnerf_render_moved", ctx.handle, io, n, S, N_importance, flags, impl, C.byref(moves.abi()), evaluated)
    else:
        ctx.call("dmnerf_render_moved_copies", ctx.handle, io, n, S, N_importance, flags, impl, C.byref(moves.abi()),
                 moves.copy_flags(), evaluated)
    out["evaluated"] = (int(evaluated[0]), int(evaluated[1]))
    return out


def _check_moved(moves, who, device, model_coarse, model_fine):
    """ValueError unless `moves` is an objects.MovedScene built on `device`; RuntimeError when the networks would record
    gradients (a moved render is inference-only)."""
    from .autograd import _needs_grad
    from .objects import MovedScene
    if not isinstance(moves, MovedScene):
        raise ValueError("%s: moves must be an objects.render_moves(...) result, got %r" % (who, type(moves).__name__))
    if moves.device != torch.device(device):
        raise ValueError("%s: the moves were built on %s, the render runs on %s" % (who, moves.device, device))
    if _needs_grad(model_coarse, model_fine):
        raise RuntimeError("%s: a scene edit (object selection, region, appearance, moves) is inference-only; call it under "
                           "torch.no_grad() or with parameters that do not require grad" % who)


class LazyRenderDict(dict):
    """Result of an inference dm_nerf() call.  The per-ray maps come from the single fused kernel; the per-sample tensors
    the reference also returns (`raw_*`, `z_vals_*`: consumed only by the training-time penalizer) are produced on
    first access (indexing, `in`, get, keys / values / items, iteration, len) by re-rendering through the stage-by-stage kernels
    with the same random draws; entries that already exist (the per-ray maps, possibly sliced by the caller) are left untouched.
    Note: the lazily produced `z_vals_fine` / `raw_fine` come from that second render; on isolated rays an importance sample may
    land in the neighbouring bin compared with the fused kernel's own fine depths (same arithmetic, different reduction order
    in the coarse weights' last bits), so they describe the same distribution but are not bit-identical to what produced the maps."""
    LAZY = ("raw_fine", "raw_coarse", "z_vals_fine", "z_vals_coarse", "weights_fine", "weights_coarse")

    def __init__(self, data, rerender):
        super().__init__(data)
        self._rerender = rerender

    def _materialise(self):
        if self._rerender is not None:
            full, self._rerender = self._rerender(), None
            for k, v in full.items():
                if not super().__contains__(k):
                    super().__setitem__(k, v)

    def __missing__(self, key):
        if key in self.LAZY and self._rerender is not None:
            self._materialise()
            return super().__getitem__(key)
        raise KeyError(key)

    def __contains__(self, key):
        return super().__contains__(key) or (key in self.LAZY and self._rerender is not None)

    def keys(self):
        self._materialise()
        return super().keys()

    def items(self):
        self._materialise()
        return super().items()

    def values(self):
        self._materialise()
        return super().values()

    def get(self, key, default=None):
        if key in self.LAZY:
            self._materialise()
        return super().get(key, default)

    def __iter__(self):
        self._materialise()
        return super().__iter__()

    def __len__(self):
        self._materialise()
        return super().__len__()


def dm_nerf(rays, position_embedder, view_embedder, model_coarse, model_fine, z_vals_coarse, args):
    """Same signature and return dict as reference networks/render.py:31-96."""
    from .autograd import _needs_grad
    _check_embedders(position_embedder, view_embedder)
    rays_o, rays_d = rays
    perturb = float(args.perturb) if args.perturb else 0.0
    if _needs_grad(model_coarse, model_fine):
        from .backward import render_rays_grad
        out = render_rays_grad(rays_o, rays_d, model_coarse, model_fine, z_vals_coarse, perturb, args.N_importance)
    else:
        # drawn once here: the lazy re-render must see the fused render's uniforms
        t_rand, u = reference_draws(perturb, rays_o.reshape(-1, 3).shape[0], z_vals_coarse.shape[-1], args.N_importance,
                                    rays_o.device)
        kw = dict(perturb=perturb, N_importance=args.N_importance, t_rand=t_rand, u=u)
        fused = render_rays(rays_o, rays_d, model_coarse, model_fine, z_vals_coarse, want_raw=False, want_samples=False, **kw)
        out = LazyRenderDict(fused, lambda: render_rays(rays_o, rays_d, model_coarse, model_fine, z_vals_coarse,
                                                        want_raw=True, **kw))
    if getattr(args, "is_train", False) and getattr(args, "N_ins", None) is not None:      # render.py:88-90
        out["ins_fine"] = out["ins_fine"][-args.N_ins:]
        out["ins_coarse"] = out["ins_coarse"][-args.N_ins:]
    return out


# north_star aliases (SURVEY.md name-mapping table)
raw2outputs = render_train


def render_frame(H, W, K, c2w, near, far, model_coarse, model_fine, N_samples=64, N_importance=128, pixel_range=None,
                 keep_all_ins=False, impl=_lib.IMPL_AUTO, device="cuda", keep_objects=None, region=None, appearance=None,
                 moves=None, chunk=8192):
    """One camera of the reference's test-time loop (render_test, networks/tester.py:55-76) through the frame entry point of
    the C ABI: rays are generated on the device from K / c2w (get_rays_k), the coarse depth row from near / far
    (z_val_sample), the pixels are rendered by the fused kernel and the maps come back as HOST tensors:
    rgb [H,W,3], ins [H,W,ins_num], depth [H,W], acc [H,W] (or [n, ...] rows when a pixel_range = (begin, count) is given --
    the per-rank slice of a sharded frame).  keep_objects, region and appearance: object selection, region selection and object
    appearance as in render_rays; impl as in render_rays.
    moves: an objects.MovedScene: the frame's rays (get_rays_k, on the device) are rendered by render_rays(moves=) in chunks of
    `chunk` rays into device maps, which return as host tensors of the same shapes; the result gains evaluated = (coarse, fine)
    targets over the frame.  `chunk` bounds the moved render's device scratch, about 190 KB per ray at ins_num 93 with 64 + 128
    samples (1.5 GB at the default 8192; DESIGN.md, "Rendering moved objects")."""
    if moves is not None:
        return _render_frame_moved(H, W, K, c2w, near, far, model_coarse, model_fine, N_samples, N_importance, pixel_range,
                                   keep_all_ins, impl, device, keep_objects, region, appearance, moves, chunk)
    impl = _lib.infer_impl(impl)
    dev = torch.device(device)
    ctx = get_context(dev)
    ins_num = bind_pair(ctx, model_coarse, model_fine)
    edit, held = scene_edit("render_frame", ins_num, torch.device("cuda", ctx.index), model_coarse, model_fine, keep_objects,
                            region, appearance)
    begin, count = (0, H * W) if pixel_range is None else (int(pixel_range[0]), int(pixel_range[1]))
    n_ins = ins_num + 1 if keep_all_ins else ins_num
    pin = dev.type == "cuda"
    out = {"rgb": torch.empty(count, 3, pin_memory=pin), "ins": torch.empty(count, n_ins, pin_memory=pin),
           "depth": torch.empty(count, pin_memory=pin), "acc": torch.empty(count, pin_memory=pin)}
    io = _lib.RenderIO(rgb_fine=_lib.ptr(out["rgb"]), ins_fine=_lib.ptr(out["ins"]), depth_fine=_lib.ptr(out["depth"]),
                       acc_fine=_lib.ptr(out["acc"]), edit=edit)
    flags = _lib.FLAG_KEEP_INS if keep_all_ins else 0
    Kf, Cf = _lib.camera(K, c2w)
    ctx.call("dmnerf_render_frame_host", ctx.handle, Kf, Cf, H, W, float(near), float(far), begin, count, N_samples,
             N_importance, flags, impl, C.byref(io))
    if pixel_range is None:
        out = {"rgb": out["rgb"].reshape(H, W, 3), "ins": out["ins"].reshape(H, W, n_ins), "depth": out["depth"].reshape(H, W),
               "acc": out["acc"].reshape(H, W)}
    return out


def frame_rays(H, W, K, c2w, near, far, N_samples, device):
    """The rays [H * W, 3] (get_rays_k on the device) and the shared coarse depth row [N_samples] (z_val_sample) of one camera."""
    from .helpers import get_rays_k, z_val_sample
    c2w = torch.as_tensor(c2w, dtype=torch.float32).to(device)
    ro, rd = get_rays_k(H, W, K, c2w)
    return ro.reshape(-1, 3), rd.reshape(-1, 3), z_val_sample(1, near, far, N_samples, device=device)[0].contiguous()


def _render_frame_moved(H, W, K, c2w, near, far, model_coarse, model_fine, N_samples, N_importance, pixel_range, keep_all_ins, impl,
                        device, keep_objects, region, appearance, moves, chunk):
    """render_frame(moves=): render_rays(moves=) over chunks of the frame's rays into preallocated device maps."""
    if isinstance(chunk, (bool,)) or int(chunk) != chunk or int(chunk) < 1:
        raise ValueError("render_frame: chunk must be an integer >= 1, got %r" % (chunk,))
    dev = torch.device(device)
    ctx = get_context(dev)
    dev = torch.device("cuda", ctx.index)
    ins_num = bind_pair(ctx, model_coarse, model_fine)
    _check_moved(moves, "render_frame", dev, model_coarse, model_fine)
    begin, count = (0, H * W) if pixel_range is None else (int(pixel_range[0]), int(pixel_range[1]))
    if not (0 <= begin and 0 <= count and begin + count <= H * W):
        raise ValueError("render_frame: pixel range [%d, +%d) outside the %dx%d frame" % (begin, count, H, W))
    ro, rd, z = frame_rays(H, W, K, c2w, near, far, N_samples, dev)
    n_ins = ins_num + 1 if keep_all_ins else ins_num
    maps = {"rgb": torch.empty(count, 3, device=dev), "ins": torch.empty(count, n_ins, device=dev),
            "depth": torch.empty(count, device=dev), "acc": torch.empty(count, device=dev)}
    evaluated = [0, 0]
    for b in range(0, count, int(chunk)):
        e = min(b + int(chunk), count)
        r = render_rays(ro[begin + b:begin + e], rd[begin + b:begin + e], model_coarse, model_fine, z, N_importance=N_importance,
                        want_raw=False, want_coarse=False, keep_all_ins=keep_all_ins, impl=impl, keep_objects=keep_objects,
                        region=region, appearance=appearance, moves=moves)
        for k in maps:
            maps[k][b:e] = r[k + "_fine"]
        evaluated = [evaluated[0] + r["evaluated"][0], evaluated[1] + r["evaluated"][1]]
    out = {k: v.cpu() for k, v in maps.items()}
    if pixel_range is None:
        out = {"rgb": out["rgb"].reshape(H, W, 3), "ins": out["ins"].reshape(H, W, n_ins), "depth": out["depth"].reshape(H, W),
               "acc": out["acc"].reshape(H, W)}
    out["evaluated"] = tuple(evaluated)
    return out
