"""GPU: data-parallel training (dmnerf_b200.distributed).  The sharded loss kernels against the unsharded ones in one process,
then train_iteration over two real processes against one process stepping the same batches, and at world 1 against the
single-GPU iteration.  Run as a script (`--worker`), this file is also the worker of the two-process test."""
import os
import subprocess
import sys
import tempfile
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from dmnerf_b200 import _lib, synth                                                # noqa: E402
from dmnerf_b200.testing import make_models, rel_l2                                # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda"
MAP_KEYS = ("rgb_coarse", "rgb_fine", "ins_coarse", "ins_fine", "depth_coarse", "depth_fine")


def _i32(t):
    return _lib.ptr(t, torch.int32)


def _rel(a, b):
    a, b = float(torch.as_tensor(a).detach()), float(torch.as_tensor(b).detach())
    return abs(a - b) / max(abs(b), 1e-30)


# ------------------------------------------------------------------------------------------------- kernels, one process
def _pieces(n, world):
    from dmnerf_b200.parallel import shard_range
    return [shard_range(n, world, r)[:2] for r in range(world)]


def _sharded_ins(ctx, pred, labels, k, pieces):
    """The sharded instance-loss kernels on `pieces` (row ranges of pred / labels), gathered by stacking."""
    n = pred.shape[0]
    bitmaps = torch.stack([torch.empty(_lib.LABEL_WORDS, device=DEV, dtype=torch.int32) for _ in pieces])
    for r, (lo, hi) in enumerate(pieces):
        ctx.call("dmnerf_ins_label_bitmap", _i32(labels[lo:hi]), hi - lo, _i32(bitmaps[r]))
    parts = torch.empty(len(pieces), 3 * k * (k + 1), device=DEV, dtype=torch.float64)
    rows, nvs = [], []
    for r, (lo, hi) in enumerate(pieces):
        gt_row = torch.empty(hi - lo, device=DEV, dtype=torch.int32)
        nv = torch.empty(1, device=DEV, dtype=torch.int32)
        ctx.call("dmnerf_ins_label_rows_merged", _i32(bitmaps), len(pieces), _i32(labels[lo:hi]), hi - lo, k, _i32(gt_row), _i32(nv))
        ctx.call("dmnerf_hungarian_partials", _lib.ptr(pred[lo:hi]), _i32(gt_row), hi - lo, k, _lib.ptr(parts[r], torch.float64))
        rows.append(gt_row); nvs.append(nv)
    e = lambda *s: torch.empty(s, device=DEV, dtype=torch.float32)
    c = {"cost_ce": e(k, k), "cost_siou": e(k, k), "tp": e(k, k), "col_sum": e(k), "row_count": e(k)}
    ctx.call("dmnerf_hungarian_costs_merged", _lib.ptr(parts, torch.float64), len(pieces), n, k, _lib.ptr(c["cost_ce"]),
             _lib.ptr(c["cost_siou"]), _lib.ptr(c["tp"]), _lib.ptr(c["col_sum"]), _lib.ptr(c["row_count"]))
    return c, rows, nvs


def _batch(n, k, seed, n_labels):
    gen = torch.Generator().manual_seed(seed)
    pred = torch.softmax(3 * torch.randn(n, k, generator=gen), -1).to(DEV).contiguous()
    ids = torch.randperm(900, generator=gen)[:n_labels] * 70 + 3                        # sparse ids in [0, 65536)
    labels = ids[torch.randint(0, n_labels - 2, (n,), generator=gen)]
    labels[:2] = ids[n_labels - 2]                                                       # in the first piece only
    labels[-1] = ids[n_labels - 1]                                                       # in the last piece only
    return pred, labels.to(torch.int32).to(DEV).contiguous()


@pytest.mark.parametrize("crop", [False, True])
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("k", [13, 93])
def test_sharded_instance_and_penalizer_kernels_match_the_one_shard_entries(k, world, crop):
    """W shards of the instance loss and the penalizer against the one-process entries (dmnerf_hungarian_costs, ins_criterion,
    emptiness_penalizer): the shards' label ranks, costs, matching, losses and gradients."""
    from dmnerf_b200.distributed import instance_rows
    from dmnerf_b200.engine import get_context
    from dmnerf_b200.evaluator import _costs, ins_criterion
    from dmnerf_b200.penalizer import emptiness_penalizer
    ctx = get_context(DEV)
    n = 1001
    n_ins = 307 if crop else None
    shards = _pieces(n, world)
    ins = [instance_rows(lo, hi, n, n_ins) for lo, hi in shards]               # global ins rows [a, b) -> rows of the labels
    pieces = [(a - off, b - off) for a, b, off in ins]
    m = n if n_ins is None else n_ins
    pred, labels = _batch(m, k, 11 + k + world, min(k, 9))
    assert sum(b - a for a, b in pieces) == m and (not crop or pieces[0][0] == pieces[0][1])     # crop: rank 0 has none
    # unsharded: label ranks, costs, assignment
    gt_row = torch.empty(m, device=DEV, dtype=torch.int32)
    nv = torch.empty(1, device=DEV, dtype=torch.int32)
    ctx.call("dmnerf_ins_label_rows", _i32(labels), m, k, _i32(gt_row), _i32(nv))
    ref = _costs(pred, gt_row)
    c, rows, nvs = _sharded_ins(ctx, pred, labels, k, pieces)
    assert torch.equal(torch.cat(rows), gt_row) and all(torch.equal(v, nv) for v in nvs)
    for key in ref:
        assert rel_l2(c[key].cpu(), ref[key].cpu()) <= 1e-6, key
    assign = []
    for cc in (ref, c):
        roc = torch.empty(k, device=DEV, dtype=torch.int32)
        l3 = torch.empty(3, device=DEV)
        ctx.call("dmnerf_hungarian_assign", _lib.ptr(cc["cost_ce"]), _lib.ptr(cc["cost_siou"]), _lib.ptr(cc["col_sum"]), _i32(nv), m, k,
                 _i32(roc), _lib.ptr(l3))
        assign.append((roc, l3))
    assert torch.equal(assign[0][0], assign[1][0])
    for j in range(3):
        assert _rel(assign[1][1][j], assign[0][1][j]) <= 1e-6
    # gradient: ins_criterion's autograd vs the concatenated shard gradients
    p = pred.clone().requires_grad_(True)
    loss, vce, ice, vsi = ins_criterion(p, labels, k)
    assert _rel(vce, assign[0][1][0]) <= 1e-6 and _rel(vsi, assign[0][1][2]) <= 1e-6
    loss.backward()
    g3 = torch.ones(3, device=DEV)
    d = torch.empty_like(pred)
    for (lo, hi), gr in zip(pieces, rows):
        ctx.call("dmnerf_ins_loss_backward", _lib.ptr(pred[lo:hi]), _i32(gr), hi - lo, m, k, _i32(assign[1][0]), _i32(nvs[0]),
                 _lib.ptr(c["tp"]), _lib.ptr(c["col_sum"]), _lib.ptr(c["row_count"]), _lib.ptr(g3), _lib.ptr(d[lo:hi]))
    assert rel_l2(d.cpu(), p.grad.cpu()) <= 1e-6
    # penalizer over the shards of the whole batch (samples of every ray)
    S, C = 40, 4 + k + 1
    gen = torch.Generator().manual_seed(k + world)
    raw = (2 * torch.randn(n, S, C, generator=gen)).to(DEV)
    z = (4.0 + 11.0 * torch.sort(torch.rand(n, S, generator=gen), -1).values).to(DEV)
    depth = (5.0 + 9.0 * torch.rand(n, 1, generator=gen)).to(DEV)
    rays_d = torch.randn(n, 3, generator=gen).to(DEV)
    r = raw.clone().requires_grad_(True)
    pen = emptiness_penalizer(r, z, depth, rays_d, 0.05, 0.05)
    pen.backward()
    head = int(ctx.lib.dmnerf_penalizer_state_bytes())
    parts = []
    shard_loss = torch.empty(1, device=DEV)
    for lo, hi in shards:
        buf = torch.empty(int(ctx.lib.dmnerf_penalizer_partials_bytes(hi - lo, S, C)), device=DEV, dtype=torch.uint8)
        ctx.call("dmnerf_penalizer_forward", _lib.ptr(raw[lo:hi]), _lib.ptr(z[lo:hi]), _lib.ptr(depth[lo:hi, 0].contiguous()),
                 _lib.ptr(rays_d[lo:hi]), hi - lo, S, C, 0.05, 0.05, _lib.ptr(buf, torch.uint8), _lib.ptr(shard_loss))
        parts.append(buf[:head])
    state = torch.empty(head, device=DEV, dtype=torch.uint8)
    ploss = torch.empty(1, device=DEV)
    ctx.call("dmnerf_penalizer_merge", _lib.ptr(torch.stack(parts), torch.uint8), world, C, _lib.ptr(state, torch.uint8),
             _lib.ptr(ploss))
    assert _rel(ploss, pen) <= 1e-6
    d_raw = torch.empty_like(raw)
    one = torch.ones(1, device=DEV)
    for lo, hi in shards:
        ctx.call("dmnerf_penalizer_backward", _lib.ptr(raw[lo:hi]), _lib.ptr(z[lo:hi]), _lib.ptr(depth[lo:hi, 0].contiguous()),
                 _lib.ptr(rays_d[lo:hi]), hi - lo, S, C, 0.05, 0.05, _lib.ptr(state, torch.uint8), _lib.ptr(one), _lib.ptr(d_raw[lo:hi]), 0)
    assert rel_l2(d_raw.cpu(), r.grad.cpu()) <= 1e-6
    ctx.sync_check()


@pytest.mark.parametrize("k", [13, 93, 128])
def test_one_process_costs_are_the_one_shard_merge_bit_for_bit(k):
    """dmnerf_hungarian_costs finalises the partials kernel's sums inside its own launch: every output equals
    dmnerf_hungarian_partials followed by dmnerf_hungarian_costs_merged at world 1, bit for bit, with unlabelled rays (row -1)
    and every ray count class of the kernel's 32-row chunks and 8 warps."""
    from dmnerf_b200.engine import get_context
    from dmnerf_b200.evaluator import _cost_buffers, _cost_ptrs, _costs
    ctx = get_context(DEV)
    for n in (1, 2, 31, 32, 33, 255, 256, 257, 1000, 2048, 3071, 3072):
        gen = torch.Generator().manual_seed(n * 131 + k)
        pred = torch.softmax(3 * torch.randn(n, k, generator=gen), -1).to(DEV).contiguous()
        gt_row = torch.randint(-1, min(k, 9), (n,), generator=gen).to(torch.int32).to(DEV)
        one = _costs(pred, gt_row)
        part = torch.empty(3 * k * (k + 1), device=DEV, dtype=torch.float64)
        ctx.call("dmnerf_hungarian_partials", _lib.ptr(pred), _i32(gt_row), n, k, _lib.ptr(part, torch.float64))
        merged = _cost_buffers(k, DEV)
        ctx.call("dmnerf_hungarian_costs_merged", _lib.ptr(part, torch.float64), 1, n, k, *_cost_ptrs(merged))
        for key in one:
            assert torch.equal(one[key], merged[key]), (n, key)


@pytest.mark.parametrize("n, s, k", [(1, 1, 13), (37, 64, 13), (300, 64, 59), (1024, 192, 93), (200, 40, 127)])
def test_penalizer_forward_is_the_one_shard_merge_bit_for_bit(n, s, k):
    """The penalizer forward's own loss and head equal dmnerf_penalizer_merge of that head at world 1, bit for bit, up to
    thousands of blocks (1024 x 192 samples at ins_num 93: 3072 block slots reduced by the last block)."""
    from dmnerf_b200.engine import get_context
    ctx = get_context(DEV)
    C = 4 + k + 1
    gen = torch.Generator().manual_seed(n + s + k)
    raw = (2 * torch.randn(n, s, C, generator=gen)).to(DEV)
    z = (4.0 + 11.0 * torch.sort(torch.rand(n, s, generator=gen), -1).values).to(DEV)
    depth = (5.0 + 9.0 * torch.rand(n, generator=gen)).to(DEV)
    rays_d = torch.randn(n, 3, generator=gen).to(DEV)
    u8 = torch.uint8
    part = torch.empty(int(ctx.lib.dmnerf_penalizer_partials_bytes(n, s, C)), device=DEV, dtype=u8)
    loss = torch.empty(1, device=DEV)
    ctx.call("dmnerf_penalizer_forward", _lib.ptr(raw), _lib.ptr(z), _lib.ptr(depth), _lib.ptr(rays_d), n, s, C, 0.05, 0.05,
             _lib.ptr(part, u8), _lib.ptr(loss))
    head = int(ctx.lib.dmnerf_penalizer_state_bytes())
    state = torch.empty(head, device=DEV, dtype=u8)
    merged = torch.empty(1, device=DEV)
    ctx.call("dmnerf_penalizer_merge", _lib.ptr(part[:head], u8), 1, C, _lib.ptr(state, u8), _lib.ptr(merged))
    assert torch.equal(loss, merged) and bool(torch.isfinite(loss).all())
    assert torch.equal(part[:32], state[:32])                   # populations and sums (the block counter is the forward's own)


def test_ins_criterion_and_its_one_process_sharded_form_agree_bit_for_bit():
    """ins_criterion and ins_criterion_sharded(..., n_global = n) in one process run the same Function: bitwise-equal losses,
    matchings and gradients."""
    from dmnerf_b200.distributed import ins_assignment_sharded, ins_criterion_sharded
    from dmnerf_b200.evaluator import ins_assignment, ins_criterion
    n, k = 3072, 93
    pred, labels = _batch(n, k, 17, 40)
    got = []
    for fn in (ins_criterion, lambda p, lab, kk: ins_criterion_sharded(p, lab, kk, n)):
        p = pred.clone().requires_grad_(True)
        parts = fn(p, labels, k)
        parts[0].backward()
        got.append(([x.detach() for x in parts], p.grad))
    for a, b in zip(got[0][0] + [got[0][1]], got[1][0] + [got[1][1]]):
        assert torch.equal(a, b)
    assert torch.equal(ins_assignment(pred, labels, k)[0], ins_assignment_sharded(pred, labels, k, n)[4])


@pytest.mark.parametrize("case", ["out_of_range", "too_many"])
def test_sharded_labels_rejected_on_every_shard_and_reported_on_the_next_call(case):
    from dmnerf_b200.distributed import ins_criterion_sharded
    from dmnerf_b200.engine import get_context
    ctx = get_context(DEV)
    ctx.lib.dmnerf_ins_status_take()
    k, n = 13, 600
    pred, labels = _batch(n, k, 5, 8)
    if case == "out_of_range":
        labels[450] = 70000                                                                  # one piece only
    else:
        labels[:300] = torch.arange(300, device=DEV, dtype=torch.int32) % 7 + 1000           # 7 + 8 distinct labels > 13
    c, rows, nvs = _sharded_ins(ctx, pred, labels, k, _pieces(n, 3))
    assert all(int(v) == -1 for v in nvs)
    assert ctx.lib.dmnerf_ins_status_take() == (701 if case == "out_of_range" else 702)
    # through the Python entry point (one process): NaN loss now, an error on the next call
    loss = ins_criterion_sharded(pred, labels, k, n)[0]
    assert torch.isnan(loss)
    with pytest.raises(RuntimeError, match="code 70"):
        ins_criterion_sharded(pred, labels, k, n)


# -------------------------------------------------------------------------------------------------------- training step
def _scene(H=48, W=64):
    wl = synth.workload("dmsr_study")
    gen = torch.Generator().manual_seed(9)
    rgb = torch.rand(H, W, 3, generator=gen).to(DEV)
    lab = (torch.arange(H * W).reshape(H, W) * 7 // (H * W)).to(torch.int16).to(DEV)
    return rgb, lab, torch.from_numpy(wl["c2w"]).float().to(DEV), synth.dmsr_intrinsics(H, W), wl


def _args(ins_num, n_ins=None):
    return types.SimpleNamespace(perturb=1.0, N_importance=128, N_samples=64, is_train=True, N_ins=n_ins, ins_num=ins_num,
                                 penalize=True, tolerance=0.05, deta_w=0.05, lrate=5e-4, lrate_decay=2, near=4.0, far=15.0)


def _make_batch(it, rgb, lab, pose, K, n, crop):
    from dmnerf_b200.helpers import get_select_crop, get_select_full
    np.random.seed(100 + it)
    if crop:
        H, W = lab.shape
        ins_index = np.nonzero((lab.reshape(-1) < 5).cpu().numpy())[0]
        crop_mask = np.ones((H, W), dtype=np.int64)
        return get_select_crop(rgb, pose, K, lab, ins_index, crop_mask, n)
    return get_select_full(rgb, pose, K, lab, n) + (None,)


def _models(ins_num):
    mc, mf, _, _ = make_models(201, 202, ins_num, DEV)
    mc.train(); mf.train()
    params = list(mc.parameters()) + list(mf.parameters())
    return mc, mf, torch.optim.Adam(params, lr=5e-4, betas=(0.9, 0.999))


def _record(res, mc, mf, out):
    from dmnerf_b200.engine import ordered_params
    params = ordered_params(mc)[0] + ordered_params(mf)[0]
    return {"maps": {k: out[k].detach().cpu() for k in MAP_KEYS},
            "row_of_col": [res["row_of_col_coarse"].cpu(), res["row_of_col_fine"].cpu()],
            "losses": {k: float(res[k].detach().sum()) for k in ("total", "rgb", "ins", "emptiness")},
            "grads": [p.grad.detach().cpu().clone() for p in params], "params": [p.detach().cpu().clone() for p in params]}


def _one_process(n, steps, ins_num, crop=False):
    """The single-GPU iteration (render.dm_nerf + evaluator + penalizer, train_dmsr.py:23-71) on the same batches."""
    from dmnerf_b200.embedder import get_embedder
    from dmnerf_b200.evaluator import img2mse, ins_assignment, ins_criterion
    from dmnerf_b200.helpers import z_val_sample
    from dmnerf_b200.penalizer import ins_penalizer
    from dmnerf_b200.render import dm_nerf
    rgb, lab, pose, K, wl = _scene()
    mc, mf, opt = _models(ins_num)
    pe, ve = get_embedder(10)[0], get_embedder(4)[0]
    zc = z_val_sample(n, 4.0, 15.0, 64, device=DEV)
    recs = []
    for it in range(steps):
        tc, ti, rays, n_ins = _make_batch(it, rgb, lab, pose, K, n, crop)
        args = _args(ins_num, n_ins)
        torch.manual_seed(it)
        info = dm_nerf(rays, pe, ve, mc, mf, zc, args)
        rgb_c, rgb_f = img2mse(info["rgb_coarse"], tc), img2mse(info["rgb_fine"], tc)
        ins_c = ins_criterion(info["ins_coarse"], ti, ins_num)
        ins_f = ins_criterion(info["ins_fine"], ti, ins_num)
        roc = [ins_assignment(info[key].detach(), ti, ins_num)[0] for key in ("ins_coarse", "ins_fine")]
        pen = ins_penalizer(info["raw_fine"], info["z_vals_fine"], info["depth_fine"], rays[1], args) \
            + ins_penalizer(info["raw_coarse"], info["z_vals_coarse"], info["depth_coarse"], rays[1], args)
        ins_loss, rgb_loss = ins_f[0] + ins_c[0], rgb_f + rgb_c
        total = ins_loss + rgb_loss + pen
        opt.zero_grad()
        total.sum().backward()
        opt.step()
        for g in opt.param_groups:
            g["lr"] = args.lrate * (0.1 ** (it / (args.lrate_decay * 1000)))
        res = {"total": total, "rgb": rgb_loss, "ins": ins_loss, "emptiness": pen, "row_of_col_coarse": roc[0],
               "row_of_col_fine": roc[1]}
        recs.append(_record(res, mc, mf, info))
    return recs


def _data_parallel(n, steps, ins_num, crop=False, group=None):
    from dmnerf_b200.distributed import replicas_identical, train_iteration
    from dmnerf_b200.engine import ordered_params
    from dmnerf_b200.helpers import z_val_sample
    rgb, lab, pose, K, wl = _scene()
    mc, mf, opt = _models(ins_num)
    zc = z_val_sample(n, 4.0, 15.0, 64, device=DEV)
    recs = []
    for it in range(steps):
        batch = _make_batch(it, rgb, lab, pose, K, n, crop)
        torch.manual_seed(it)
        res = train_iteration(it, batch, mc, mf, opt, _args(ins_num, batch[3]), zc, group=group)
        rec = _record(res, mc, mf, res["out"])
        rec["lo"], rec["hi"] = res["lo"], res["hi"]
        rec["identical"] = replicas_identical(ordered_params(mc)[0] + ordered_params(mf)[0], group)
        recs.append(rec)
    return recs


def _compare(dp_ranks, ref, crop=False):
    """dp_ranks: per rank, the records of its steps; ref: the one-process records.  The one-process comparison is made at
    step 0, where both start from equal parameters.  Later steps start from parameters that already differ by the Adam-step
    difference (Adam scales each gradient element by its own magnitude, so an element whose gradient is within the dW rounding
    of zero can move the other way: 2.3e-5 relative L2 measured on an H100), and the two trajectories drift apart (the first
    layer's gradients, ~1e-8, by 1.8e-3 at step 1 and 1.1e-2 at step 2); there only the replicas' agreement is checked."""
    r = ref[0]
    for rank_recs in dp_ranks:
        d = rank_recs[0]
        lo, hi = d["lo"], d["hi"]
        for k in MAP_KEYS:
            if crop and k.startswith("ins"):
                continue                                       # the one-process maps are cut to the last N_ins rays
            assert torch.equal(d["maps"][k], r["maps"][k][lo:hi]), k       # rays are independent in the kernels
        for a, b in zip(d["row_of_col"], r["row_of_col"]):
            assert torch.equal(a, b)
        for k, v in r["losses"].items():
            assert _rel(d["losses"][k], v) <= 1e-5, (k, d["losses"][k], v)
        for j, (a, b) in enumerate(zip(d["grads"], r["grads"])):
            assert rel_l2(a, b) <= 2e-4, (j, rel_l2(a, b))
        for j, (a, b) in enumerate(zip(d["params"], r["params"])):
            assert rel_l2(a, b) <= 1e-4, (j, rel_l2(a, b))
    for it in range(len(ref)):                                 # replicas bit-identical after every step
        for x in dp_ranks:
            assert x[it]["identical"]
            assert torch.equal(x[it]["row_of_col"][0], dp_ranks[0][it]["row_of_col"][0])
            assert all(torch.equal(p, q) for p, q in zip(x[it]["params"], dp_ranks[0][it]["params"])), it


@pytest.mark.parametrize("crop", [False, True])
def test_world_one_train_iteration_equals_the_single_gpu_iteration(crop):
    ref = _one_process(1024, 2, 13, crop)
    dp = _data_parallel(1024, 2, 13, crop)
    _compare([dp], ref, crop)


def _spawn_world_two(n, steps, ins_num, tmp):
    store = os.path.join(tmp, "store")
    procs = []
    env = dict(os.environ)
    try:
        for rank in range(2):
            out = os.path.join(tmp, "rank%d.pt" % rank)
            procs.append(subprocess.Popen([sys.executable, os.path.abspath(__file__), "--worker", str(rank), "2", store, out, str(n),
                                           str(steps), str(ins_num)], env=env))
        for p in procs:
            assert p.wait(timeout=600) == 0
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
                p.wait()
    return [torch.load(os.path.join(tmp, "rank%d.pt" % r)) for r in range(2)]


@pytest.mark.parametrize("n", [3072, 1023])
def test_world_two_train_iteration_equals_one_process(n):
    steps = 3
    with tempfile.TemporaryDirectory() as tmp:
        dp = _spawn_world_two(n, steps, 13, tmp)
    ref = _one_process(n, steps, 13)
    _compare(dp, ref)
    assert dp[0][0]["hi"] == dp[1][0]["lo"] and dp[1][0]["hi"] == n
    if n == 3072:                                                   # bit-reproducible run to run at a fixed world size
        with tempfile.TemporaryDirectory() as tmp:
            again = _spawn_world_two(n, steps, 13, tmp)
        for a, b in zip(dp, again):
            for ra, rb in zip(a, b):
                assert all(torch.equal(x, y) for x, y in zip(ra["grads"] + ra["params"], rb["grads"] + rb["params"]))
                assert ra["losses"] == rb["losses"]


def _worker(rank, world, store, out, n, steps, ins_num):
    import torch.distributed as dist
    two_gpus = torch.cuda.device_count() >= world
    torch.cuda.set_device(rank if two_gpus else 0)
    global DEV
    DEV = "cuda:%d" % torch.cuda.current_device()
    dist.init_process_group("nccl" if two_gpus else "gloo", init_method="file://" + store, rank=rank, world_size=world)
    try:
        recs = _data_parallel(n, steps, ins_num, group=None)
        torch.save(recs, out)
    finally:
        dist.destroy_process_group()


if __name__ == "__main__" and len(sys.argv) > 1 and sys.argv[1] == "--worker":
    _worker(*[int(a) if a.isdigit() else a for a in sys.argv[2:]])
