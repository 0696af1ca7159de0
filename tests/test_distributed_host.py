"""CPU: the arithmetic of data-parallel training (dmnerf_b200.distributed) that needs no device: row and crop ranges, the
full-size draws every rank slices, the colour loss at world size 1, and the C ABI of the sharded losses."""
import os
import re

import pytest
import torch

from dmnerf_b200 import _lib
from dmnerf_b200.distributed import img2mse_sharded, instance_rows
from dmnerf_b200.parallel import shard_range, world_of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("n", [1, 7, 1023, 1024, 3072])
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_shards_tile_the_batch_in_rank_order(n, world):
    ranges = [shard_range(n, world, r)[:2] for r in range(world)]
    assert ranges[0][0] == 0 and ranges[-1][1] == n
    assert all(a[1] == b[0] for a, b in zip(ranges, ranges[1:]))
    assert all(lo <= hi for lo, hi in ranges)


@pytest.mark.parametrize("n_ins", [None, 0, 1, 307, 921, 1023])
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_instance_rows_are_each_shards_part_of_the_last_n_ins_rays(n_ins, world):
    n = 1023
    m = n if n_ins is None else n_ins
    got = []
    for r in range(world):
        lo, hi, _ = shard_range(n, world, r)
        a, b, off = instance_rows(lo, hi, n, n_ins)
        assert lo <= a <= b == hi and off == n - m
        assert set(range(a, b)) == set(range(lo, hi)) & set(range(n - m, n))
        got += list(range(a - off, b - off))
    assert got == list(range(m))                              # the label rows, in order, each on one rank


def test_every_rank_slices_the_same_full_size_uniforms():
    """train_iteration draws torch.rand([N, 64]) then torch.rand([N, 128]) at full size on every rank: the ranks' rows put
    together are the one-process draws, and the second draw does not depend on the world size."""
    n = 1023
    torch.manual_seed(5)
    t_ref, u_ref = torch.rand(n, 64), torch.rand(n, 128)
    for world in (2, 3, 8):
        ts, us = [], []
        for r in range(world):
            torch.manual_seed(5)
            t, u = torch.rand(n, 64), torch.rand(n, 128)
            lo, hi, _ = shard_range(n, world, r)
            ts.append(t[lo:hi]); us.append(u[lo:hi])
        assert torch.equal(torch.cat(ts), t_ref) and torch.equal(torch.cat(us), u_ref)


def test_colour_loss_at_world_one_is_img2mse_with_its_gradient():
    assert world_of() == (1, 0)
    gen = torch.Generator().manual_seed(2)
    x = torch.rand(300, 3, generator=gen, dtype=torch.float32).requires_grad_(True)
    y = torch.rand(300, 3, generator=gen)
    x2 = x.detach().clone().requires_grad_(True)
    got = img2mse_sharded(x, y, 300)
    want = torch.mean((x2 - y) ** 2)
    assert abs(float(got) - float(want)) <= 1e-6 * float(want)
    got.backward(); want.backward()
    assert torch.allclose(x.grad, x2.grad, rtol=1e-5, atol=1e-9)


def test_loss_entry_points_are_declared_and_bound_and_the_removed_ones_are_gone():
    header = open(os.path.join(ROOT, "include", "dmnerf_b200.h")).read()
    names = ["dmnerf_ins_label_bitmap", "dmnerf_ins_label_rows_merged", "dmnerf_hungarian_partials", "dmnerf_hungarian_costs_merged",
             "dmnerf_ins_loss_backward", "dmnerf_penalizer_partials_bytes", "dmnerf_penalizer_forward", "dmnerf_penalizer_merge"]
    for name in names:
        assert re.search(r"DMNERF_API\s+[\w\s\*]+?\b%s\s*\(" % name, header), name
        assert name in _lib.PROTOTYPES, name
    assert re.search(r"#define DMNERF_LABEL_WORDS %d\b" % _lib.LABEL_WORDS, header)
    # n and n_global of the shard's backward are both 64-bit
    assert _lib.PROTOTYPES["dmnerf_ins_loss_backward"][1][2:4] == [_lib.C.c_int64, _lib.C.c_int64]
    for gone in ("dmnerf_ins_loss_backward_dev", "dmnerf_ins_loss_backward_shard", "dmnerf_penalizer_partials"):
        assert gone not in _lib.PROTOTYPES and not re.search(r"\b%s\s*\(" % gone, header), gone
