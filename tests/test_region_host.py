"""CPU checks of region selection (DESIGN.md, "Region selection"): the fp32 voxel map against the sweep's own grid points, its
rounding, the builders' argument checks and label words, the render_objects tool's flags, and the oracles' per-sample exclusion
defaulting to their results without one."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from dmnerf_b200 import objects as OB  # noqa: E402
from dmnerf_b200 import synth  # noqa: E402
from oracle import dmnerf_f16 as H  # noqa: E402
from oracle import dmnerf_oracle as O  # noqa: E402
from oracle import inventory_oracle as IO  # noqa: E402
from oracle import objects_oracle as OO  # noqa: E402
from oracle import region_oracle as RO  # noqa: E402


def transforms():
    """Non-trivial scene transforms: a rotation about a tilted axis with an offset, and a cyclic permutation."""
    a = 0.7
    c, s = np.cos(a), np.sin(a)
    R1 = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]) @ np.array([[1, 0, 0], [0, np.cos(0.3), -np.sin(0.3)], [0, np.sin(0.3), np.cos(0.3)]])
    T1 = np.eye(4)
    T1[:3, :3], T1[:3, 3] = R1, [0.31, -1.7, 2.2]
    T2 = np.eye(4)
    T2[:3, :3], T2[:3, 3] = np.array([[0, 0, 1], [1, 0, 0], [0, 1, 0]]), [-0.5, 0.25, 1.0]
    return [(T1, (1.9, 7.0, 7.0)), (T2, (3.0, 2.5, 4.0))]


@pytest.mark.parametrize("dim", [64, 97, 256])
def test_voxel_map_sends_every_grid_point_to_its_index(dim):
    for T, ext in transforms():
        A, b = OB.grid_affine(T, dim, ext)
        vm = OB.voxel_map(T, dim, ext)
        assert vm.dtype == np.float32 and np.array_equal(vm, RO.voxel_map(A, b))
        n = dim ** 3
        for start in range(0, n, 1 << 21):
            v = np.arange(start, min(n, start + (1 << 21)), dtype=np.int64)
            idx = np.stack([v // (dim * dim), (v // dim) % dim, v % dim], -1)
            pts = IO.grid_points_fp32(idx, T, dim, ext)
            got = RO.voxel_of(vm, pts)
            assert np.array_equal(got.astype(np.int64), idx), (dim, start)


def test_half_index_points_round_to_even_and_non_finite_points_are_outside():
    vm = np.concatenate([np.eye(3), np.zeros((3, 1))], 1).astype(np.float32)
    k = np.arange(-3, 12, dtype=np.float32)
    pts = np.stack([k + 0.5, np.full_like(k, 2.0), np.full_like(k, 3.0)], -1)
    assert np.array_equal(RO.voxel_of(vm, pts)[:, 0], np.rint(k + 0.5))
    assert np.array_equal(RO.voxel_of(vm, pts)[:, 0] % 2, np.zeros_like(k))            # half to even, never half up
    dim = 8
    bits = RO.pack(np.ones((dim, dim, dim), dtype=bool))
    look = RO.lookup(vm, bits, dim, pts)
    inside = (np.rint(k + 0.5) >= 0) & (np.rint(k + 0.5) <= dim - 1)
    assert np.array_equal(look == 1, inside) and np.array_equal(look == -1, ~inside)
    bad = np.array([[np.nan, 1, 1], [1, np.inf, 1], [1, 1, -np.inf], [7.4, 7.4, 7.4], [7.6, 0, 0], [-0.6, 0, 0]], dtype=np.float32)
    assert RO.lookup(vm, bits, dim, bad).tolist() == [-1, -1, -1, 1, -1, -1]


def test_pack_and_unpack_and_dilation_twin():
    rng = np.random.default_rng(5)
    for dim in (5, 9):
        m = rng.random((dim, dim, dim)) < 0.1
        w = RO.pack(m)
        assert w.shape[0] == (dim ** 3 + 31) // 32 and np.array_equal(RO.unpack(w, dim), m)
        tail = dim ** 3 % 32
        if tail:
            assert int(w[-1]) >> tail == 0
    one = np.zeros((6, 6, 6), dtype=bool)
    one[0, 0, 5] = True
    d6, d26 = RO.dilate(one, 1, 6), RO.dilate(one, 1, 26)
    assert d6.sum() == 4 and d26.sum() == 8 and not d26[0, 1, 0] and not d26[5, 0, 5]     # no wrap across a face
    assert np.array_equal(RO.dilate(one, 0), one)


def test_builder_arguments_and_label_words():
    assert OB.label_words([0, 31, 32, 127]) == [1 | (1 << 31), 1, 0, 1 << 31]
    with pytest.raises(ValueError):
        OB.label_words([128])
    grid = torch.zeros(4, 4, 4, dtype=torch.int32)
    cc = {"grid": grid, "label": np.zeros(1, dtype=np.int16), "voxels": np.ones(1, dtype=np.int64)}
    T = np.eye(4)
    for kw in ({"dilate": -1}, {"dilate": 1.5}, {"connectivity": 18}, {"outside": "maybe"}):
        with pytest.raises(ValueError):
            OB.component_region(cc, [0], T, **kw)
        with pytest.raises(ValueError):
            OB.region_from_mask(grid.bool(), T, **kw)
    with pytest.raises(RuntimeError, match="CUDA"):                        # a host grid: no CPU fallback
        OB.component_region(cc, [0], T)
    vm = OB.voxel_map(T, 4)
    good = 2
    for bits, dim in ((torch.zeros(good, dtype=torch.int32), 4),          # host tensor
                      (torch.zeros(good, dtype=torch.int64), 4), (torch.zeros(good + 1, dtype=torch.int32), 4),
                      (torch.zeros(good, dtype=torch.int32), 1), (torch.zeros(good, dtype=torch.int32), 1291)):
        with pytest.raises(ValueError):
            OB.Region(bits, dim, vm)
    with pytest.raises(ValueError):
        bad = vm.copy()
        bad[0, 0] = np.nan
        OB.Region(torch.zeros(good, dtype=torch.int32), 4, bad)


class _Fake:
    """A Region whose bits are not checked (the words logic only)."""
    applies_words = OB.Region.applies_words

    def __init__(self, applies):
        self.applies = applies


def test_applies_words_default_to_every_label():
    assert _Fake(None).applies_words(13) == [(1 << 14) - 1, 0, 0, 0]
    assert _Fake(None).applies_words(93) == [0xFFFFFFFF, 0xFFFFFFFF, (1 << 30) - 1, 0]
    assert _Fake([5, 0, 0, 0]).applies_words(13) == [5, 0, 0, 0]


def _tool():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import render_objects
    return render_objects


BASE = ["ck.tar", "--pose", "p.npy", "--hwk", "48", "64"] + ["1"] * 9 + ["--out", "d"]


def test_render_objects_tool_flags():
    R = _tool()
    a = R.parse(BASE + ["--keep", "1", "2"])
    assert (a.keep, a.remove, a.region, a.H, a.W) == ([1, 2], None, None, 48, 64)
    assert (a.near, a.far, a.N_samples, a.N_importance) == (4.0, 15.0, 64, 128)
    a = R.parse(BASE + ["--remove", "3"])
    assert (a.keep, a.remove, a.region) == (None, [3], None)
    a = R.parse(BASE + ["--no-floaters", "--transform", "t.txt"])
    assert (a.keep, a.remove, a.region, a.dilate, a.connectivity, a.grid_dim, a.level) == (None, None, "no_floaters", 1, 26, 256, 0.45)
    a = R.parse(BASE + ["--keep", "2", "--keep-piece", "7", "9", "--transform", "t.txt", "--dilate", "0", "--connectivity", "6"])
    assert (a.keep, a.region, a.keep_piece, a.dilate, a.connectivity) == ([2], "keep", [7, 9], 0, 6)
    a = R.parse(BASE + ["--drop-piece", "4", "--transform", "t.txt", "--extents", "2", "3", "4", "--grid-dim", "128"])
    assert (a.region, a.drop_piece, a.extents, a.grid_dim) == ("drop", [4], [2.0, 3.0, 4.0], 128)
    for bad in ([], ["--keep", "1", "--remove", "2"], ["--no-floaters"], ["--no-floaters", "--drop-piece", "1", "--transform", "t"],
                ["--keep-piece", "1", "--transform", "t", "--dilate", "-1"], ["--no-floaters", "--transform", "t", "--connectivity", "8"]):
        with pytest.raises(SystemExit):
            R.parse(BASE + bad)


def test_oracle_exclusion_defaults_to_the_result_without_one():
    """region_oracle.render / render_on_depths without an exclusion (or with one that excludes nothing) are objects_oracle.render
    and dmnerf_f16.render_on_depths bit for bit; excluding every sample empties the maps as the empty selection does."""
    wl = synth.workload("dmsr_study")
    sel = np.linspace(0, wl["H"] * wl["W"] - 1, 24).astype(np.int64)
    ro, rd = torch.from_numpy(wl["rays_o"][sel]).double(), torch.from_numpy(wl["rays_d"][sel]).double()
    wc, wf = synth.make_weights(101, wl["ins_num"]), synth.make_weights(202, wl["ins_num"])
    p64c, p64f = O.to_torch(wc, torch.float64), O.to_torch(wf, torch.float64)
    z = O.z_val_sample(24, wl["near"], wl["far"], 64, dtype=torch.float64)
    keep = torch.ones(wl["ins_num"] + 1, dtype=torch.bool)
    keep[3] = False
    nothing = lambda zz, lab: torch.zeros(lab.shape, dtype=torch.bool)      # noqa: E731
    ref = OO.render(ro, rd, p64c, p64f, z, keep)
    for got in (RO.render(ro, rd, p64c, p64f, z, keep), RO.render(ro, rd, p64c, p64f, z, keep, exclude=nothing)):
        assert sorted(got) == sorted(ref)
        for k in ref:
            assert torch.equal(ref[k], got[k]), k
    net_c, net_f = (lambda x: O.mlp_forward(p64c, x)), (lambda x: O.mlp_forward(p64f, x))
    for sel_ in (None, keep):
        t0 = H.render_on_depths(net_c, net_f, ro, rd, ref["z_vals_coarse"], ref["z_vals_fine"], fp32_inputs=False, keep=sel_)
        for ex in (None, nothing):
            t1 = RO.render_on_depths(net_c, net_f, ro, rd, ref["z_vals_coarse"], ref["z_vals_fine"], fp32_inputs=False, keep=sel_,
                                     exclude=ex)
            assert sorted(t0) == sorted(t1)
            for k in t0:
                assert torch.equal(t0[k], t1[k]), k
    allx = RO.render(ro, rd, p64c, p64f, z, keep, exclude=lambda zz, lab: torch.ones(lab.shape, dtype=torch.bool))
    assert bool((allx["acc_fine"] == 0).all()) and bool((allx["ins_fine"] == 0.5).all())
    # the region exclusion of an empty grid that keeps its outside and applies to no label excludes nothing
    T, ext = transforms()[0]
    dim = 16
    ex = RO.exclusion(OB.voxel_map(T, dim, ext), RO.pack(np.zeros((dim,) * 3, dtype=bool)), dim, [0, 0, 0, 0], True,
                      ro.float().numpy(), rd.float().numpy())
    assert not bool(ex(ref["z_vals_fine"], OO.object_labels(ref["raw_fine"])).any())
