"""GPU: rendering moved objects per sample (dmnerf_render_moved, render_rays(moves=), render_frame(moves=)) -- identity and absent
moves against the unedited stage render, the edited raw against the rule applied by torch to the device network
(oracle/render_moves_oracle.py), solid samples against edited_sweep's grid, composition with selection and appearance, the frame
driver against the ray entry point and the frame entry point, manipulation_transform moves against the fp64 oracle, an
arrangement's moves, tools/move_objects.py --render samples, and the host-side rejections."""
import ctypes as C

import numpy as np
import pytest
import torch

from dmnerf_b200 import _lib
from dmnerf_b200 import objects as OB
from dmnerf_b200.autograd import mlp_forward_points, mlp_forward_rays
from dmnerf_b200.engine import get_context
from dmnerf_b200.render import frame_rays, render_frame, render_rays
from dmnerf_b200.testing import make_models
from oracle import dmnerf_oracle as O
from oracle import render_moves_oracle as RM

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NEAR, FAR, NI = 4.0, 15.0, 128
VOXEL = np.float32((FAR - NEAR) / NI)
EXT = (4.0, 4.0, 4.0)
T = np.eye(4)
MAPS = ("rgb_fine", "ins_fine", "depth_fine", "acc_fine", "weights_fine", "z_vals_fine", "rgb_coarse", "ins_coarse", "depth_coarse",
        "acc_coarse", "weights_coarse", "z_vals_coarse", "raw_coarse", "raw_fine")


@pytest.fixture(scope="module", params=[13, 93])
def nets(request):
    nc, nf, _, _ = make_models(101, 202, request.param, DEV)
    return nc, nf, request.param


@pytest.fixture(scope="module")
def twins(nets):
    """A coarse and a fine network with the same weights: the coarse pass then sees what edited_sweep sees."""
    _, _, ins_num = nets
    nc, nf, _, _ = make_models(303, 303, ins_num, DEV)
    return nc, nf, ins_num


def _sweep(nf, dim):
    ins_num = int(nf.ins_linear.weight.shape[0]) - 1
    return OB.occupancy_objects(nf, T, OB.object_mask(ins_num, remove=[]), dim, EXT, NEAR, FAR, NI, device=DEV)


def _level(occ):
    x = occ.flatten().float()
    x = x[x > 0]
    return float(x.kthvalue(max(1, int(0.5 * x.numel()))).values)


def _top_labels(occ, labels, lv, n):
    lab = labels[occ > lv].cpu().numpy()
    k, c = np.unique(lab, return_counts=True)
    return [int(x) for x in k[np.argsort(-c, kind="stable")][:n]]


def _rays(n, seed=0):
    """Rays from a sphere of radius 3 towards points inside the grid, and the coarse depths 1 .. 5."""
    g = torch.Generator().manual_seed(seed)
    o = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1) * 3.0
    d = (torch.rand(n, 3, generator=g) - 0.5) * 2.0 - o
    return o.to(DEV), d.to(DEV), torch.linspace(1.0, 5.0, 64).to(DEV)


def _translate(v):
    m = np.eye(4)
    m[:3, 3] = v
    return m


def _quarter_turn_z(c):
    R = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    m = np.eye(4)
    m[:3, :3] = R
    m[:3, 3] = np.asarray(c) - R @ np.asarray(c)
    return m


@pytest.fixture(scope="module")
def scene(nets):
    nc, nf, ins_num = nets
    with torch.no_grad():
        occ, labels = _sweep(nf, 64)
    lv = _level(occ)
    return dict(occ=occ, labels=labels, level=lv, solid=_top_labels(occ, labels, lv, 3))


def _same(a, b, keys=MAPS):
    for k in keys:
        assert torch.equal(a[k], b[k]), k


# ---- 1, 2: identity and absent moves ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("impl", [_lib.IMPL_UMMA, _lib.IMPL_UMMA_F16])
@pytest.mark.parametrize("with_piece", [False, True])
def test_identity_move_is_the_unedited_render_bit_for_bit(nets, scene, impl, with_piece):
    nc, nf, ins_num = nets
    mv = scene["solid"][0]
    pieces = None
    if with_piece:
        pieces = [OB.region_from_mask(torch.ones((64,) * 3, dtype=torch.bool, device=DEV), T, EXT, applies=[mv])]
    moved = OB.render_moves(scene["occ"], scene["labels"], T, [(mv, np.eye(4))], EXT, scene["level"], NEAR, FAR, NI,
                            pieces=pieces)
    o, d, z = _rays(512)
    with torch.no_grad():
        ref = render_rays(o, d, nc, nf, z, want_raw=True, impl=impl)
        got = render_rays(o, d, nc, nf, z, want_raw=True, impl=impl, moves=moved)
    assert got["evaluated"][0] > 0 and got["evaluated"][1] > 0
    _same(got, ref)


def test_absent_label_and_empty_box_change_nothing(nets, scene):
    nc, nf, ins_num = nets
    present = set(int(k) for k in torch.unique(scene["labels"][scene["occ"] > scene["level"]]).cpu().tolist())
    absent = next(k for k in range(ins_num + 1) if k not in present)
    o, d, z = _rays(512, 1)
    with torch.no_grad():
        ref = render_rays(o, d, nc, nf, z, want_raw=True)
        for moves, boxes in (([(absent, _translate([0.5, 0.0, 0.0]))], None),
                             ([(scene["solid"][0], _translate([0.5, 0.0, 0.0]))], [OB.EMPTY_BOX])):
            moved = OB.render_moves(scene["occ"], scene["labels"], T, moves, EXT, scene["level"], NEAR, FAR, NI, boxes=boxes)
            got = render_rays(o, d, nc, nf, z, want_raw=True, moves=moved)
            assert got["evaluated"] == (0, 0)
            _same(got, ref)


# ---- 3: the edited raw against the rule applied by torch --------------------------------------------------------------------------

def _axis_rays():
    """Rays along the network x axis through every grid line's origin, depths 0 .. 4 in steps of 0.125: the coarse samples are the
    grid points of the dim 33 grid of extents 4, all exact in fp32."""
    ys = np.arange(-2.0, 2.01, 0.125)
    o = torch.tensor([[-2.0, y, zz] for y in ys for zz in ys], dtype=torch.float32, device=DEV)
    d = torch.tensor([[1.0, 0.0, 0.0]], device=DEV).expand_as(o).contiguous()
    return o, d, torch.arange(0.0, 4.0 + 1e-6, 0.125, dtype=torch.float32, device=DEV)


def _device_evaluate(model):
    def f(t, dirs):
        return mlp_forward_points(model, torch.from_numpy(t).to(DEV), torch.from_numpy(dirs).to(DEV), impl=_lib.IMPL_UMMA)
    return f


@pytest.mark.parametrize("kind", ["translation", "quarter_turn"])
def test_edited_raw_is_the_rule_on_the_device_network(nets, kind):
    nc, nf, ins_num = nets
    with torch.no_grad():
        occ, labels = _sweep(nf, 33)
    lv = _level(occ)
    mv = _top_labels(occ, labels, lv, 1)[0]
    trans = _translate([0.25, -0.125, 0.0]) if kind == "translation" else _quarter_turn_z([0.125, -0.25, 0.0])
    moved = OB.render_moves(occ, labels, T, [(mv, trans)], EXT, lv, NEAR, FAR, NI)
    o, d, z = _axis_rays()
    with torch.no_grad():
        got = render_rays(o, d, nc, nf, z, want_raw=True, moves=moved)
        raw_c = mlp_forward_rays(nc, o, d, z.expand(o.shape[0], -1).contiguous())
        raw_f = mlp_forward_rays(nf, o, d, got["z_vals_fine"])
    move = [dict(label=mv, trans=trans, box=moved.boxes[0], piece=None, rest_drop=False)]
    want_c, ev_c = RM.apply_moves(raw_c, o, d, z.expand(o.shape[0], -1), move, T, EXT, 33, _device_evaluate(nc), lv, VOXEL)
    want_f, ev_f = RM.apply_moves(raw_f, o, d, got["z_vals_fine"], move, T, EXT, 33, _device_evaluate(nf), lv, VOXEL)
    assert torch.equal(got["raw_coarse"], want_c)
    assert torch.equal(got["raw_fine"], want_f)
    assert got["evaluated"] == (ev_c, ev_f) and ev_c > 0
    # the sweep (and so mv) comes from the fine network: the move changes the fine pass at least
    assert not (torch.equal(want_c, raw_c) and torch.equal(want_f, raw_f))


# ---- 4: solid samples against edited_sweep's grid ---------------------------------------------------------------------------------

def _labels_for(occ, labels, n):
    """A level (a quantile of the positive occupancies) at which the sweep has at least n solid labels, and n of them."""
    for q in (0.5, 0.3, 0.15, 0.05):
        x = occ.flatten().float()
        x = x[x > 0]
        lv = float(x.kthvalue(max(1, int(q * x.numel()))).values)
        mvs = _top_labels(occ, labels, lv, n)
        if len(mvs) == n:
            return lv, mvs
    pytest.skip("the synthetic sweep has fewer than %d solid labels" % n)


def _half_piece(occ, labels, lv, mv, dim):
    """The piece of mv's solid points below the median of their first grid index (the rest is the other half)."""
    solid = (labels == mv) & (occ > lv)
    i = torch.nonzero(solid)[:, 0].float()
    mask = solid.clone()
    mask[int(i.median()) + 1:] = False
    return OB.region_from_mask(mask, T, EXT, applies=[mv])


@pytest.mark.parametrize("case", ["1", "3", "piece_keep", "piece_drop"])
def test_solid_samples_equal_the_edited_sweep_on_grid_points(twins, case):
    nc, nf, ins_num = twins
    n_moves = 3 if case == "3" else 1
    with torch.no_grad():
        occ, labels = _sweep(nf, 33)
    lv, mvs = _labels_for(occ, labels, n_moves)
    assert len(mvs) == n_moves
    shifts = ([0.25, 0.0, 0.0], [0.0, -0.125, 0.0], [0.0, 0.0, 0.375])
    moves = [(k, _translate(s)) for k, s in zip(mvs, shifts)]
    pieces, rest = None, "keep"
    if case.startswith("piece"):
        pieces, rest = [_half_piece(occ, labels, lv, mvs[0], 33)], case[6:]
    with torch.no_grad():
        e_occ, e_lab = OB.edited_sweep(nf, T, moves, 33, EXT, lv, NEAR, FAR, NI, pieces=pieces, rest=rest)
        moved = OB.render_moves(occ, labels, T, moves, EXT, lv, NEAR, FAR, NI, pieces=pieces, rest=rest)
        o, d, z = _axis_rays()
        got = render_rays(o, d, nc, nf, z, want_raw=True, moves=moved)
    raw = got["raw_coarse"]
    solid = (RM.occupancy(raw[..., 3], VOXEL) > lv).cpu().numpy()
    lab = torch.argmax(torch.sigmoid(raw[..., 4:]), -1).cpu().numpy()
    # sample (ray, s) is grid point i = s (x = -2 + 0.125 s), and network (y, z) = (-2 l_k, 2 l_j)
    on = o.cpu().numpy()
    j = np.rint((on[:, 2] + 2.0) * 8).astype(int)
    k = np.rint((2.0 - on[:, 1]) * 8).astype(int)
    g_solid = (e_occ > lv).cpu().numpy()[:, j, k].T
    g_lab = e_lab.cpu().numpy()[:, j, k].T
    assert np.array_equal(solid, g_solid)
    assert np.array_equal(lab[solid], g_lab[g_solid])
    u_solid = (occ > lv).cpu().numpy()[:, j, k].T
    assert not np.array_equal(g_solid, u_solid)                       # the edit changed the solid set


# ---- 5: manipulation_transform moves against the fp64 oracle, teacher-forced ------------------------------------------------------
FLOOR = 0.1                                                           # of each map's scale, as test_gpu_appearance
AMBIGUOUS_CAP = 0.01                                                  # of the rays


def _centre(occ, labels, lv, mv, dim):
    A, b = OB.grid_affine(T, dim, EXT)
    idx = torch.nonzero((labels == mv) & (occ > lv)).double().mean(0).cpu().numpy()
    return A @ idx + b


@pytest.mark.parametrize("mode", ["rotation", "scale", "multi_moves"])
def test_manipulation_moves_against_the_fp64_oracle(nets, scene, mode):
    """manipulation_transform moves (a 90 degree yaw, a 1.2 scale, or a yaw on one label with a scale-rotate-translate on another):
    the edited raw of both passes equals the rule on the device network bit for bit (the scaled and turned view directions
    included), and every map and weight is within 1e-4 (floor: a tenth of the map's scale) of the fp64 network and composite on
    the kernel's own depths.  A ray is set aside only where the fp64 decisions differ from the device's (a label or an occupancy
    tied at the level to fp32 precision): at most 1 % of the rays."""
    nc, nf, ins_num = nets
    _, _, wc, wf = make_models(101, 202, ins_num, DEV)
    occ, labels, lv = scene["occ"], scene["labels"], scene["level"]
    mvs = scene["solid"]
    spec = {"rotation": [(mvs[0], "rotation")], "scale": [(mvs[0], "scale")],
            "multi_moves": [(mvs[0], "rotation"), (mvs[1 % len(mvs)], "multi")]}[mode]
    moves = [(k, np.asarray(OB.manipulation_transform(_centre(occ, labels, lv, k, 64), m)["transformations"][0]["transformation"]))
             for k, m in spec]
    moved = OB.render_moves(occ, labels, T, moves, EXT, lv, NEAR, FAR, NI)
    om = [dict(label=k, trans=m, box=moved.boxes[i], piece=None, rest_drop=False) for i, (k, m) in enumerate(moves)]
    o, d, z = _rays(513, 4)
    with torch.no_grad():
        got = render_rays(o, d, nc, nf, z, want_raw=True, moves=moved)
        zc, zf = got["z_vals_coarse"], got["z_vals_fine"]
        rec32 = {"coarse": [], "fine": []}
        for tag, net, zz in (("coarse", nc, zc), ("fine", nf, zf)):
            raw32 = mlp_forward_rays(net, o, d, zz)
            want, ev = RM.apply_moves(raw32, o, d, zz, om, T, EXT, 64, _device_evaluate(net), lv, VOXEL, rec32[tag])
            assert torch.equal(got["raw_" + tag], want), tag
            assert got["evaluated"][0 if tag == "coarse" else 1] == ev
        p64 = [{k: v.to(DEV) for k, v in O.to_torch(w, torch.float64).items()} for w in (wc, wf)]
        rec64 = {}
        ref = RM.render_on_depths(o, d, p64[0], p64[1], zc, zf, om, T, EXT, 64, lv, VOXEL, rec64)
    n = o.shape[0]
    aside = np.zeros(n, dtype=bool)
    for tag, s in (("coarse", zc.shape[1]), ("fine", zf.shape[1])):
        for (t32, v32), (t64, v64) in zip(rec32[tag], rec64[tag]):
            aside |= ((t32 != t64) | (v32 != v64)).reshape(n, s).any(-1)
    assert aside.sum() <= AMBIGUOUS_CAP * n, int(aside.sum())
    assert got["evaluated"][0] > 0
    keep = torch.from_numpy(~aside).to(DEV)
    for tag in ("coarse", "fine"):
        for m in ("rgb", "depth", "acc", "ins", "weights"):
            g, r = got[m + "_" + tag].double()[keep], ref[m + "_" + tag][keep]
            scale = float(r.abs().max())
            err = float(((g - r).abs() / torch.clamp(r.abs(), min=FLOOR * scale)).max())
            assert err <= 1e-4, (tag, m, err)


# ---- 6: composition ---------------------------------------------------------------------------------------------------------------

def test_moves_compose_with_selection_and_appearance(nets, scene):
    nc, nf, ins_num = nets
    mv = scene["solid"][0]
    moved = OB.render_moves(scene["occ"], scene["labels"], T, [(mv, _translate([0.3, 0.2, 0.0]))], EXT, scene["level"], NEAR, FAR, NI)
    o, d, z = _rays(512, 2)
    geometry = ("weights_fine", "depth_fine", "acc_fine", "ins_fine", "weights_coarse", "depth_coarse", "acc_coarse", "ins_coarse")
    with torch.no_grad():
        base = render_rays(o, d, nc, nf, z, want_raw=True, moves=moved)
        tinted = render_rays(o, d, nc, nf, z, want_raw=True, moves=moved, appearance=OB.Appearance(ins_num, colour={mv: OB.tint((1, 0, 0))}))
        _same(tinted, base, geometry)
        assert not torch.equal(tinted["rgb_fine"], base["rgb_fine"])
        only = render_rays(o, d, nc, nf, z, want_raw=True, moves=moved, keep_objects=[mv])
        lab = torch.argmax(torch.sigmoid(only["raw_fine"][..., 4:]), -1)
        assert torch.all(only["weights_fine"][lab != mv] == 0)
        gone = render_rays(o, d, nc, nf, z, want_raw=True, moves=moved, appearance=OB.Appearance(ins_num, density={mv: 0.0}))
        unselected = render_rays(o, d, nc, nf, z, want_raw=True, moves=moved, keep_objects=[k for k in range(ins_num + 1) if k != mv])
        _same(gone, unselected, geometry + ("rgb_fine",))


def test_a_floater_region_composes_with_the_moves(nets, scene):
    """A region that drops the moved label's samples in one half of the grid, tested at each sample's own point with the edited
    labels: the edited raw is the region-free moved render's (coarse bit for bit), and each pass's maps are the composite of the
    kernel's own edited raw with exactly the region's samples dropped (fp32 torch composite, 1e-5)."""
    from oracle import objects_oracle as OO
    from oracle import region_oracle as RO
    nc, nf, ins_num = nets
    mv = scene["solid"][0]
    moved = OB.render_moves(scene["occ"], scene["labels"], T, [(mv, _translate([0.3, 0.2, 0.0]))], EXT, scene["level"], NEAR, FAR, NI)
    half = torch.zeros((64,) * 3, dtype=torch.bool, device=DEV)
    half[:32] = True
    region = OB.region_from_mask(half, T, EXT, applies=[mv])
    o, d, z = _rays(512, 5)
    with torch.no_grad():
        free = render_rays(o, d, nc, nf, z, want_raw=True, moves=moved)
        got = render_rays(o, d, nc, nf, z, want_raw=True, moves=moved, region=region)
    assert torch.equal(got["raw_coarse"], free["raw_coarse"])
    excl = RO.exclusion(region.voxel_map, region.bits.cpu().numpy(), 64, region.applies_words(ins_num), True, o.cpu().numpy(),
                        d.cpu().numpy())
    dropped = 0
    for tag in ("coarse", "fine"):
        raw, zz = got["raw_" + tag], got["z_vals_" + tag]
        ex = excl(zz, OO.object_labels(raw))
        dropped += int(ex.sum())
        rgb, w, depth, ins, acc = O.composite(RO.exclude_samples(raw, ex), zz, d)
        for m, want in (("rgb", rgb), ("weights", w), ("depth", depth), ("ins", ins), ("acc", acc)):
            assert float((got[m + "_" + tag] - want).abs().max()) <= 1e-5 * max(1.0, float(want.abs().max())), (tag, m)
    assert dropped > 0


# ---- 7: the frame driver ----------------------------------------------------------------------------------------------------------

def test_render_frame_equals_render_rays_on_the_frame_rays(nets, scene):
    from dmnerf_b200 import synth
    nc, nf, ins_num = nets
    w = synth.workload("dmsr_study")
    H, W = 96, 128
    mv = scene["solid"][0]
    moved = OB.render_moves(scene["occ"], scene["labels"], T, [(mv, _translate([0.3, 0.2, 0.0]))], EXT, scene["level"], NEAR, FAR, NI)
    c2w = torch.as_tensor(w["c2w"], dtype=torch.float32)
    with torch.no_grad():
        ro, rd, z = frame_rays(H, W, w["K"], c2w, w["near"], w["far"], 64, torch.device(DEV))
        ref = render_rays(ro, rd, nc, nf, z, want_raw=False, want_coarse=False, moves=moved)
        for chunk in (4096, 8192):
            fr = render_frame(H, W, w["K"], c2w, w["near"], w["far"], nc, nf, moves=moved, chunk=chunk, device=DEV)
            for k in ("rgb", "ins", "depth", "acc"):
                assert torch.equal(fr[k].reshape(H * W, -1).squeeze(-1), ref[k + "_fine"].cpu()), (chunk, k)
            assert fr["evaluated"] == ref["evaluated"]
        part = render_frame(H, W, w["K"], c2w, w["near"], w["far"], nc, nf, moves=moved, chunk=4096, pixel_range=(1000, 5000),
                            device=DEV)
        for k in ("rgb", "ins", "depth", "acc"):
            assert torch.equal(part[k].reshape(5000, -1).squeeze(-1), ref[k + "_fine"][1000:6000].cpu()), k


def test_identity_moved_frame_is_the_frame_entry_points_stage_render(nets, scene):
    """The rays and depths of render_frame(moves=) are those of the frame entry point (dmnerf_render_frame_host, forced onto the
    stage kernels by asking for raw_coarse): an identity move gives its maps and coarse depths bit for bit."""
    from dmnerf_b200 import synth
    from dmnerf_b200.render import bind_pair
    nc, nf, ins_num = nets
    w = synth.workload("dmsr_study")
    H, W = 48, 64
    mv = scene["solid"][0]
    moved = OB.render_moves(scene["occ"], scene["labels"], T, [(mv, np.eye(4))], EXT, scene["level"], NEAR, FAR, NI)
    c2w = torch.as_tensor(w["c2w"], dtype=torch.float32)
    ctx = get_context(DEV)
    n, C_ = H * W, 4 + ins_num + 1
    host = {"rgb": torch.empty(n, 3).pin_memory(), "ins": torch.empty(n, ins_num).pin_memory(), "depth": torch.empty(n).pin_memory(),
            "acc": torch.empty(n).pin_memory(), "z": torch.empty(n, 64).pin_memory(), "raw": torch.empty(n, 64, C_).pin_memory()}
    with torch.no_grad():
        got = render_frame(H, W, w["K"], c2w, w["near"], w["far"], nc, nf, moves=moved, device=DEV)
        bind_pair(ctx, nc, nf)
        io = _lib.RenderIO(rgb_fine=_lib.ptr(host["rgb"]), ins_fine=_lib.ptr(host["ins"]), depth_fine=_lib.ptr(host["depth"]),
                           acc_fine=_lib.ptr(host["acc"]), z_vals_coarse=_lib.ptr(host["z"]), raw_coarse=_lib.ptr(host["raw"]))
        Kf, Cf = _lib.camera(w["K"], c2w)
        ctx.call("dmnerf_render_frame_host", ctx.handle, Kf, Cf, H, W, float(w["near"]), float(w["far"]), 0, n, 64, NI, 0,
                 _lib.IMPL_AUTO, C.byref(io))
        _, _, z = frame_rays(H, W, w["K"], c2w, w["near"], w["far"], 64, torch.device(DEV))
    assert got["evaluated"][1] >= 0
    assert torch.equal(host["z"], z.cpu().expand(n, -1))
    for k in ("rgb", "ins", "depth", "acc"):
        assert torch.equal(got[k].reshape(n, -1).squeeze(-1), host[k]), k


# ---- 8: an arrangement's moves ----------------------------------------------------------------------------------------------------

def test_an_arrangement_renders_by_the_rule(nets):
    """arrange_objects' moves, pieces and rest, unchanged, through render_moves: the edited coarse and fine raw equal the rule
    (pieces included) on the device network, bit for bit."""
    from oracle import edit_sweep_oracle as ES
    nc, nf, ins_num = nets
    dim = 33
    with torch.no_grad():
        occ, lab = _sweep(nf, dim)
    x = occ.flatten()
    x = x[x > 0]
    lv = float(x.kthvalue(max(1, int(0.99 * x.numel()))).values)
    labels = _top_labels(occ, lab, lv, 4)
    A, b = OB.grid_affine(T, dim, EXT)
    aims = [A @ np.array([j, dim // 2, k], dtype=np.float64) + b for j, k in ((8, 8), (8, 24), (24, 8), (24, 24))]

    def cube(label):
        _, _, centre = OB._object_extent((lab == label) & (occ > lv))
        lo = [min(max(int(c) - dim // 8, 0), dim - dim // 4) for c in centre]
        m = torch.zeros((dim,) * 3, dtype=torch.bool, device=DEV)
        m[lo[0]:lo[0] + dim // 4, lo[1]:lo[1] + dim // 4, lo[2]:lo[2] + dim // 4] = True
        return OB.region_from_mask(m, T, EXT, applies=[label], outside="drop")
    items = [{"label": k, "near": x, "turns": 4, "stable": False, "piece": cube(k), "rest": "drop"} for k, x in zip(labels, aims)]
    r = OB.arrange_objects(occ, lab, T, items, (0.0, -1.0, 0.0), EXT, lv)
    if not r["moves"]:
        pytest.skip("no piece of this synthetic sweep rests on anything at level %g" % lv)
    moved = OB.render_moves(occ, lab, T, r["moves"], EXT, lv, NEAR, FAR, NI, pieces=r["pieces"], rest=r["rest"])
    om = [dict(label=k, trans=np.asarray(m), box=moved.boxes[i], rest_drop=rr == "drop",
               piece=None if pc is None else ES.Piece(pc.bits.cpu().numpy(), pc.dim, pc.voxel_map, pc.outside == "keep"))
          for i, ((k, m), pc, rr) in enumerate(zip(r["moves"], r["pieces"], r["rest"]))]
    o, d, z = _axis_rays()
    with torch.no_grad():
        got = render_rays(o, d, nc, nf, z, want_raw=True, moves=moved)
        for tag, net, zz in (("coarse", nc, z.expand(o.shape[0], -1).contiguous()), ("fine", nf, got["z_vals_fine"])):
            want, ev = RM.apply_moves(mlp_forward_rays(net, o, d, zz), o, d, zz, om, T, EXT, dim, _device_evaluate(net), lv, VOXEL)
            assert torch.equal(got["raw_" + tag], want), tag
            assert got["evaluated"][0 if tag == "coarse" else 1] == ev


def test_move_objects_render_samples_with_arrange(nets, tmp_path):
    """tools/move_objects.py --render samples --arrange on a small frame writes its PNGs and a record with render and evaluated;
    the default still renders with the exchanger."""
    import json
    import os
    import subprocess
    import sys
    nc, nf, ins_num = nets
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    dim = 33
    ck = tmp_path / "ck.tar"
    torch.save({"network_coarse_state_dict": {k: v.cpu() for k, v in nc.state_dict().items()},
                "network_fine_state_dict": {k: v.cpu() for k, v in nf.state_dict().items()}}, str(ck))
    np.save(str(tmp_path / "pose.npy"), np.eye(4, dtype=np.float32)[:3])
    np.save(str(tmp_path / "T.npy"), T)
    with torch.no_grad():
        occ, lab = _sweep(nf, dim)
    lv = _level(occ)
    labels = sorted({k for k in _top_labels(occ, lab, lv, 6) if k != ins_num})[:2]
    A, b = OB.grid_affine(T, dim, EXT)
    spec = [{"label": k, "near": (A @ np.array([16.0, j, 16.0]) + b).tolist(), "turns": 2, "any_stability": True}
            for k, j in zip(labels, (8.0, 24.0))]
    (tmp_path / "spec.json").write_text(json.dumps(spec))
    recs = {}
    for render in ("samples", None):
        out = tmp_path / ("out_%s" % render)
        cmd = [sys.executable, os.path.join(root, "tools", "move_objects.py"), str(ck), "--pose", str(tmp_path / "pose.npy"), "--hwk",
               "8", "8", "10", "0", "4", "0", "10", "4", "0", "0", "1", "--transform", str(tmp_path / "T.npy"), "--extents", "4", "4",
               "4", "--grid-dim", str(dim), "--level", str(lv), "--arrange", str(tmp_path / "spec.json"), "--down", "0", "-1", "0",
               "--dilate", "0", "--out", str(out), "--N-test", "64"] + ([] if render is None else ["--render", render])
        r = subprocess.run(cmd, capture_output=True, text=True, cwd=root)
        assert r.returncode == 0, r.stderr[-2000:]
        assert os.path.exists(out / "rgb.png") and os.path.exists(out / "instance.png")
        recs[render] = json.loads(open(out / "transform.json").read())
    s, e = recs["samples"], recs[None]
    assert s["render"] == "samples" and len(s["evaluated"]) == 2 and all(v >= 0 for v in s["evaluated"])
    assert e["render"] == "exchanger" and e["evaluated"] is None
    assert s["transformations"] == e["transformations"] and s["labels"] == e["labels"]


# ---- 9: host-side rejections ------------------------------------------------------------------------------------------------------

def test_library_rejects_before_any_launch(nets, scene):
    nc, nf, ins_num = nets
    ctx = get_context(DEV)
    from dmnerf_b200.render import bind_pair
    bind_pair(ctx, nc, nf)
    mv = scene["solid"][0]
    moved = OB.render_moves(scene["occ"], scene["labels"], T, [(mv, np.eye(4))], EXT, scene["level"], NEAR, FAR, NI)
    o, d, z = _rays(8)
    out = torch.empty(8, 3, device=DEV)
    io = _lib.RenderIO(rays_o=_lib.ptr(o), rays_d=_lib.ptr(d), z_coarse=_lib.ptr(z), rgb_fine=_lib.ptr(out))

    def call(desc, n=8, impl=_lib.IMPL_UMMA):
        ev = (C.c_int64 * 2)(-1, -1)
        torch.cuda.synchronize()
        before = _lib.launch_count()
        rc = ctx.lib.dmnerf_render_moved(ctx.handle, C.byref(io), n, 64, NI, 0, impl, C.byref(desc), ev, ctx.stream())
        assert rc != 0 and _lib.launch_count() == before and tuple(ev) == (0, 0)
        return ctx.lib.dmnerf_last_error().decode()

    def edited(**kw):
        src = moved.abi()
        d2 = _lib.RenderMoves()
        C.memmove(C.byref(d2), C.byref(src), C.sizeof(d2))
        mvs = (_lib.EditMove * 9)()
        for i in range(9):
            C.memmove(C.byref(mvs[i]), C.byref(src.moves[0]), C.sizeof(_lib.EditMove))
        for k, v in kw.items():
            if k.startswith("m_"):
                setattr(mvs[0], k[2:], v)
            else:
                setattr(d2, k, v)
        d2.moves = C.cast(mvs, C.POINTER(_lib.EditMove))
        edited.keep = mvs
        return d2

    assert "DMNERF_IMPL_SIMT" in call(edited(), impl=_lib.IMPL_SIMT)
    assert "between 1 and 8 moves" in call(edited(n_moves=9))
    assert "label %d outside" % (ins_num + 1) in call(edited(m_label=ins_num + 1))
    bad = edited()
    bad.moves[0].trans[0] = float("nan")
    assert "not finite" in call(bad)
    bad = edited()
    bad.moves[0].trans[0] = -1.0
    assert "det" in call(bad)
    bad = edited()
    bad.moves[0].box[0], bad.moves[0].box[1] = 5, 4
    assert "inverted or outside the grid" in call(bad)
    assert "level" in call(edited(level=1.0))
    assert "voxel" in call(edited(voxel=0.0))
    assert "voxel" in call(edited(voxel=float("inf")))
    piece = OB.region_from_mask(torch.ones((64,) * 3, dtype=torch.bool, device=DEV), T, EXT, applies=[(mv + 1) % (ins_num + 1)])
    bad = edited()
    bad.moves[0].piece = piece.abi(ins_num)
    assert "applies" in call(bad) or "among" in call(bad)
    assert "2^31" in call(edited(), n=(1 << 31) // (64 + NI) + 1)
