"""CPU checks of object appearance (DESIGN.md, "Object appearance"): the table builder's checks and packing, tint on grey inputs,
the oracle's consequences of the rule (no appearance and the identity table are the region oracle bit for bit, density 0 is the
exclusion of those labels, a colour-only appearance touches rgb alone), and the render_objects tool's new flags."""
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
from oracle import appearance_oracle as AO  # noqa: E402
from oracle import dmnerf_oracle as O  # noqa: E402
from oracle import objects_oracle as OO  # noqa: E402
from oracle import region_oracle as RO  # noqa: E402

IDENTITY_ROW = [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 1, 0, 0, 0]


def test_builder_packs_rows_and_defaults_to_identity():
    a = OB.Appearance(13)
    assert a.table.dtype == np.float32 and a.table.shape == (14, 16)
    assert (a.table == np.array(IDENTITY_ROW, dtype=np.float32)).all()
    m34 = np.arange(12, dtype=np.float64).reshape(3, 4) / 7.0
    m33 = np.array([[0.5, 0.25, 0.0], [0.0, 2.0, 0.0], [-1.0, 0.0, 1.0]])
    a = OB.Appearance(93, colour={0: m34, 93: m33}, density={5: 0.3, 93: 0, 7: 2.5})
    assert a.table.shape == (94, 16)
    assert np.array_equal(a.table[0, :12], m34.astype(np.float32).reshape(12)) and a.table[0, 12] == 1.0
    assert np.array_equal(a.table[93, :12], np.concatenate([m33, np.zeros((3, 1))], 1).astype(np.float32).reshape(12))
    assert a.table[93, 12] == 0.0 and a.table[5, 12] == np.float32(0.3) and a.table[7, 12] == 2.5
    assert (a.table[:, 13:] == 0).all()
    untouched = [k for k in range(94) if k not in (0, 5, 7, 93)]
    assert (a.table[untouched] == np.array(IDENTITY_ROW, dtype=np.float32)).all()


@pytest.mark.parametrize("kw", [
    {"ins_num": 0}, {"ins_num": 128},
    {"colour": {14: np.eye(3)}}, {"colour": {-1: np.eye(3)}}, {"colour": {1.5: np.eye(3)}}, {"colour": {True: np.eye(3)}},
    {"colour": {2: np.eye(4)}}, {"colour": {2: np.ones(12)}}, {"colour": {2: [[np.nan, 0, 0], [0, 1, 0], [0, 0, 1]]}},
    {"colour": {2: np.full((3, 4), 1e39)}},
    {"density": {3: -0.5}}, {"density": {3: float("nan")}}, {"density": {3: float("inf")}}, {"density": {20: 1.0}},
])
def test_builder_rejects(kw):
    kw = dict(kw)
    ins_num = kw.pop("ins_num", 13)
    with pytest.raises(ValueError):
        OB.Appearance(ins_num, **kw)


def test_tint_keeps_grey_shading():
    for rgb in ((1.0, 1.0, 1.0), (0.9, 0.1, 0.2), (0.0, 0.5, 1.0)):
        m = OB.tint(rgb)
        assert m.shape == (3, 4) and (m[:, 3] == 0).all()
        for g in (0.0, 0.25, 0.7, 1.0):
            c = np.full(3, g)
            assert np.allclose(m[:, :3] @ c, np.asarray(rgb) * g, atol=1e-12)
    grey = OB.tint((1, 1, 1))
    assert np.allclose(grey[:, :3].sum(1), 1.0) and (grey[0] == grey[1]).all() and (grey[1] == grey[2]).all()
    # a sample's colour under tint((1, 1, 1)) is its luma in every channel, through the oracle's fp32 arithmetic
    tab = OB.Appearance(1, colour={0: grey}).table
    raw = torch.randn(200, 6)
    c = AO.edited_colour(raw, torch.zeros(200, dtype=torch.long), tab)
    assert torch.equal(c[:, 0], c[:, 1]) and torch.equal(c[:, 1], c[:, 2])
    luma = torch.sigmoid(raw[:, :3]) @ torch.tensor([0.299, 0.587, 0.114])
    assert float((c[:, 0] - luma).abs().max()) < 1e-6
    for bad in ((1, 1), (1, 1, float("nan")), "red"):
        with pytest.raises(ValueError):
            OB.tint(bad)


def _scene(n=24):
    wl = synth.workload("dmsr_study")
    sel = np.linspace(0, wl["H"] * wl["W"] - 1, n).astype(np.int64)
    ro, rd = torch.from_numpy(wl["rays_o"][sel]).double(), torch.from_numpy(wl["rays_d"][sel]).double()
    wc, wf = synth.make_weights(101, wl["ins_num"]), synth.make_weights(202, wl["ins_num"])
    p64c, p64f = O.to_torch(wc, torch.float64), O.to_torch(wf, torch.float64)
    z = O.z_val_sample(n, wl["near"], wl["far"], 64, dtype=torch.float64)
    return wl["ins_num"], ro, rd, p64c, p64f, z


def _same(a, b, keys=None):
    assert sorted(a) == sorted(b)
    for k in (keys or a):
        assert torch.equal(a[k], b[k]), k


def test_oracle_without_an_appearance_and_with_the_identity_is_the_region_oracle():
    ins_num, ro, rd, pc, pf, z = _scene()
    keep = torch.ones(ins_num + 1, dtype=torch.bool)
    keep[3] = False
    ident = OB.Appearance(ins_num)
    some = lambda zz, lab: (lab % 4 == 1)                                  # noqa: E731  an exclusion that drops samples
    for sel in (None, keep):
        for ex in (None, some):
            ref = RO.render(ro, rd, pc, pf, z, sel, exclude=ex)
            _same(ref, AO.render(ro, rd, pc, pf, z, sel, exclude=ex))
            _same(ref, AO.render(ro, rd, pc, pf, z, sel, exclude=ex, appearance=ident))
            _same(ref, AO.render(ro, rd, pc, pf, z, sel, exclude=ex, appearance=ident.table))
    ref = RO.render(ro, rd, pc, pf, z, keep)
    net_c, net_f = (lambda x: O.mlp_forward(pc, x)), (lambda x: O.mlp_forward(pf, x))
    for sel in (None, keep):
        t0 = RO.render_on_depths(net_c, net_f, ro, rd, ref["z_vals_coarse"], ref["z_vals_fine"], fp32_inputs=False, keep=sel)
        for app in (None, ident):
            _same(t0, AO.render_on_depths(net_c, net_f, ro, rd, ref["z_vals_coarse"], ref["z_vals_fine"], fp32_inputs=False,
                                          keep=sel, appearance=app))


def test_density_zero_is_the_exclusion_of_those_labels():
    ins_num, ro, rd, pc, pf, z = _scene()
    gone = [1, 4, 13]
    app = OB.Appearance(ins_num, density={k: 0.0 for k in gone})
    drop = lambda zz, lab: torch.isin(lab, torch.tensor(gone))             # noqa: E731
    keep = torch.ones(ins_num + 1, dtype=torch.bool)
    keep[gone] = False
    ref = RO.render(ro, rd, pc, pf, z, keep)
    _same(ref, AO.render(ro, rd, pc, pf, z, None, exclude=drop))          # the exclusion is the selection, as a check
    _same(ref, AO.render(ro, rd, pc, pf, z, None, appearance=app))
    keep2 = keep.clone()
    keep2[2] = False
    _same(RO.render(ro, rd, pc, pf, z, keep2), AO.render(ro, rd, pc, pf, z, keep2, appearance=app))


def test_colour_only_touches_rgb_alone():
    ins_num, ro, rd, pc, pf, z = _scene()
    colour = {k: OB.tint((0.9, 0.2, 0.1)) for k in range(0, ins_num + 1, 2)}
    colour[1] = np.array([[0.0, 0.0, 1.0, 0.1], [0.0, 1.0, 0.0, -0.2], [1.0, 0.0, 0.0, 0.0]])
    app = OB.Appearance(ins_num, colour=colour)
    keep = torch.ones(ins_num + 1, dtype=torch.bool)
    keep[5] = False
    for sel in (None, keep):
        ref = RO.render(ro, rd, pc, pf, z, sel)
        got = AO.render(ro, rd, pc, pf, z, sel, appearance=app)
        _same(ref, got, [k for k in ref if not k.startswith("rgb_")])
        for p in ("coarse", "fine"):
            assert not torch.equal(ref["rgb_" + p], got["rgb_" + p])
            lab = OO.object_labels(got["raw_" + p])
            c = AO.edited_colour(got["raw_" + p], lab, app)
            assert bool(((c >= 0) & (c <= 1)).all())
            want = torch.einsum("ns,nsc->nc", got["weights_" + p], c)
            assert float((want - got["rgb_" + p]).abs().max()) < 1e-12


def test_density_scale_thickens_and_fades():
    ins_num, ro, rd, pc, pf, z = _scene()
    base = AO.render(ro, rd, pc, pf, z, None)
    lab = OO.object_labels(base["raw_coarse"])
    thick = AO.render(ro, rd, pc, pf, z, None, appearance=OB.Appearance(ins_num, density={k: 3.0 for k in range(ins_num + 1)}))
    ghost = AO.render(ro, rd, pc, pf, z, None, appearance=OB.Appearance(ins_num, density={k: 0.1 for k in range(ins_num + 1)}))
    assert lab.numel() > 0
    # on the shared coarse depths the first sample's alpha grows and shrinks with the scale
    w0 = lambda r: r["weights_coarse"][:, 0]                               # noqa: E731
    live = w0(base) > 1e-6
    assert bool(live.any())
    assert bool((w0(thick)[live] >= w0(base)[live]).all()) and bool((w0(ghost)[live] <= w0(base)[live]).all())
    assert bool((w0(thick)[live] > w0(base)[live]).any()) and bool((w0(ghost)[live] < w0(base)[live]).any())


def _tool():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import render_objects
    return render_objects


BASE = ["ck.tar", "--pose", "p.npy", "--hwk", "48", "64"] + ["1"] * 9 + ["--out", "d"]


def test_render_objects_tool_appearance_flags():
    R = _tool()
    a = R.parse(BASE + ["--keep", "1"])
    assert (a.tint, a.opacity) == ({}, {})
    a = R.parse(BASE + ["--tint", "3", "1", "0", "0"])
    assert (a.keep, a.remove, a.region, a.tint, a.opacity) == (None, None, None, {3: (1.0, 0.0, 0.0)}, {})
    a = R.parse(BASE + ["--opacity", "2", "0.3", "--opacity", "5", "0"])
    assert (a.tint, a.opacity) == ({}, {2: 0.3, 5: 0.0})
    a = R.parse(BASE + ["--remove", "4", "--tint", "1", "0.2", "0.4", "0.6", "--tint", "2", "1", "1", "1", "--opacity", "1", "2"])
    assert (a.remove, a.tint, a.opacity) == ([4], {1: (0.2, 0.4, 0.6), 2: (1.0, 1.0, 1.0)}, {1: 2.0})
    a = R.parse(BASE + ["--no-floaters", "--transform", "t.txt", "--opacity", "0", "1.5"])
    assert (a.region, a.opacity) == ("no_floaters", {0: 1.5})
    for bad in (["--tint", "1", "1", "1"], ["--tint", "1.5", "1", "1", "1"], ["--opacity", "1"], ["--opacity", "1", "-0.5"],
                ["--opacity", "1", "nan"], ["--opacity", "0.5", "1"]):
        with pytest.raises(SystemExit):
            R.parse(BASE + bad)
