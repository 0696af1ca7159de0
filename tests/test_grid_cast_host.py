"""CPU: the ray cast through a labelled grid (DESIGN.md, "Viewing the labelled grid") as oracle/grid_cast_oracle.py restates it, on
analytic grids with known answers -- exact entry times of boxes, sphere depths within a voxel diagonal, the tie rule at corners and
faces, rays that start inside a solid or are clipped by near / far, misses and degenerate directions, the keep mask, a rotated
anisotropic grid -- and the Python layer's argument checks, which run before any device work."""
import numpy as np
import pytest
import torch

from dmnerf_b200 import objects as OB
from oracle import edit_sweep_oracle as E
from oracle import grid_cast_oracle as G

DIM = 17
EXT = (DIM - 1.0,) * 3                        # one network unit per voxel
C = (DIM - 1) / 2.0                           # the grid centre's index


def _net(i, j, k):
    """The network point of index (i, j, k) with T = I and EXT: (i - c, -(k - c), j - c)."""
    return np.array([i - C, -(k - C), j - C], dtype=np.float32)


def _ndir(di, dj, dk):
    return np.array([di, -dk, dj], dtype=np.float32)


def _grid(boxes, dim=DIM):
    occ = np.zeros((dim,) * 3, dtype=np.float32)
    lab = np.zeros((dim,) * 3, dtype=np.int16)
    for (i0, i1, j0, j1, k0, k1), l in boxes:
        occ[i0:i1 + 1, j0:j1 + 1, k0:k1 + 1] = 1.0
        lab[i0:i1 + 1, j0:j1 + 1, k0:k1 + 1] = l
    return occ, lab


def _cast(occ, lab, o, d, near=0.0, far=100.0, T=np.eye(4), ext=EXT, **kw):
    return G.cast(occ, lab, T, ext, np.atleast_2d(o), np.atleast_2d(d), near, far, **kw)


def test_index_map_is_the_one_of_the_edit_oracle():
    inv, b = E.grid_index_map(np.eye(4), EXT, DIM)
    for ijk in ((0, 0, 0), (3, 5, 7), (16, 2, 9)):
        u = inv @ (_net(*ijk).astype(np.float64) - b)
        assert np.array_equal(u, np.asarray(ijk, dtype=np.float64))


@pytest.mark.parametrize("scale", [1.0, 2.0, 0.5])
def test_box_entry_times_are_exact(scale):
    occ, lab = _grid([((5, 9, 6, 10, 4, 12), 3)])
    rays = [((-10, 8, 8), (1, 0, 0), 5 - 0.5 + 10), ((30, 7, 7), (-1, 0, 0), 30 - 9.5),
            ((6, -4, 5), (0, 1, 0), 6 - 0.5 + 4), ((7, 8, 40), (0, 0, -1), 40 - 12.5)]
    for src, dij, t in rays:
        r = _cast(occ, lab, _net(*src), _ndir(*dij) * np.float32(scale))
        assert r["t"][0] == np.float32(t / scale), (src, dij, r["t"])
        assert r["label"][0] == 3
        hit = np.unravel_index(int(r["voxel"][0]), occ.shape)
        assert occ[hit] == 1.0
        # the normal of a box face is the face's: the gradient there points along the ray's axis
        n = r["normal"][0]
        expect = -_ndir(*dij).astype(np.float64)
        assert np.allclose(n, expect / np.linalg.norm(expect), atol=1e-12)


def test_sphere_depth_within_a_voxel_diagonal():
    dim, rad = 33, 9.3
    idx = np.indices((dim,) * 3).transpose(1, 2, 3, 0).astype(np.float64)
    cen = np.array([16.2, 15.7, 16.4])
    occ = (np.linalg.norm(idx - cen, axis=-1) <= rad).astype(np.float32)
    lab = np.full(occ.shape, 4, dtype=np.int16)
    ext = (dim - 1.0,) * 3
    c = (dim - 1) / 2.0
    rng = np.random.default_rng(3)
    n = 400
    dirs = rng.normal(size=(n, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    aim = cen + rng.uniform(-5, 5, size=(n, 3))
    src = aim - 40 * dirs                                             # index space
    to_net = lambda v: np.stack([v[:, 0], -v[:, 2], v[:, 1]], -1)     # noqa: E731 (index offsets -> network)
    o = to_net(src - c).astype(np.float32)
    d = to_net(dirs).astype(np.float32)
    r = G.cast(occ, lab, np.eye(4), ext, o, d, 0.0, 200.0)
    # analytic intersection in index space (o and d as the fp32 rays give them)
    so = np.stack([o[:, 0], o[:, 2], -o[:, 1]], -1).astype(np.float64) + c
    sd = np.stack([d[:, 0], d[:, 2], -d[:, 1]], -1).astype(np.float64)
    oc = so - cen
    bq = (oc * sd).sum(1)
    disc = bq * bq - ((oc * oc).sum(1) - rad * rad)
    through = disc > 1.0                                              # rays that cross well inside the sphere
    t_a = -bq - np.sqrt(np.maximum(disc, 0))
    assert through.sum() > 100
    assert (r["voxel"][through] >= 0).all()
    assert np.abs(r["t"][through] - t_a[through]).max() <= np.sqrt(3.0)
    assert (r["label"][through] == 4).all()
    # normals of a sphere point away from its centre
    hp = so + r["t"][:, None].astype(np.float64) * sd
    nidx = np.stack([r["normal"][:, 0], r["normal"][:, 2], -r["normal"][:, 1]], -1)
    out = ((hp - cen) * nidx).sum(1)
    assert (out[through] > 0).all()


def test_corner_ties_step_i_before_j_before_k():
    # from the centre of voxel (0, 0, 5) along index (1, 1, 0): the ray meets the corner of (0, 0), (1, 0), (0, 1), (1, 1)
    # exactly and steps i first, so it visits (1, 0, 5) and never (0, 1, 5)
    o, d = _net(0, 0, 5), _ndir(1, 1, 0)
    occ, lab = _grid([((1, 1, 0, 0, 5, 5), 1)])
    r = _cast(occ, lab, o, d)
    assert r["voxel"][0] == np.ravel_multi_index((1, 0, 5), occ.shape) and r["t"][0] == np.float32(0.5)
    occ, lab = _grid([((0, 0, 1, 1, 5, 5), 2)])
    assert _cast(occ, lab, o, d)["voxel"][0] == -1
    # j before k
    o, d = _net(5, 0, 0), _ndir(0, 1, 1)
    occ, lab = _grid([((5, 5, 1, 1, 0, 0), 1)])
    assert _cast(occ, lab, o, d)["voxel"][0] == np.ravel_multi_index((5, 1, 0), occ.shape)
    occ, lab = _grid([((5, 5, 0, 0, 1, 1), 1)])
    assert _cast(occ, lab, o, d)["voxel"][0] == -1


def test_a_ray_along_a_face_walks_the_upper_voxels():
    # u_j = 0.5 exactly, w_j = 0: the start voxel is floor(0.5 + 0.5) = 1
    o = _net(-3, 0.5, 4)
    d = _ndir(1, 0, 0)
    occ, lab = _grid([((6, 6, 1, 1, 4, 4), 7)])
    r = _cast(occ, lab, o, d)
    assert r["voxel"][0] == np.ravel_multi_index((6, 1, 4), occ.shape) and r["t"][0] == np.float32(8.5)
    occ, lab = _grid([((6, 6, 0, 0, 4, 4), 7)])
    assert _cast(occ, lab, o, d)["voxel"][0] == -1


def test_start_inside_a_solid_and_near_far_clipping():
    occ, lab = _grid([((4, 12, 4, 12, 4, 12), 5)])
    o, d = _net(8, 8, 8), _ndir(1, 0, 0)
    r = _cast(occ, lab, o, d, near=0.0)
    assert r["t"][0] == 0.0 and r["start_inside"][0]
    assert np.allclose(r["normal"][0], -d / np.linalg.norm(d))          # no gradient inside the block: -d
    r = _cast(occ, lab, o, d, near=2.25)
    assert r["t"][0] == np.float32(2.25) and r["voxel"][0] == np.ravel_multi_index((10, 8, 8), occ.shape)
    # from outside: far before the box is a miss, far on its face a hit
    o = _net(-4, 8, 8)
    assert _cast(occ, lab, o, d, far=7.4)["voxel"][0] == -1
    assert _cast(occ, lab, o, d, far=7.5)["t"][0] == np.float32(7.5)
    # near past the box's far side: the ray starts beyond it
    assert _cast(occ, lab, o, d, near=17.0)["voxel"][0] == -1


def test_misses_and_degenerate_directions():
    occ, lab = _grid([((0, 16, 0, 16, 0, 16), 1)])
    o = np.array([[40, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0], [0, 40, 0], [np.nan, 0, 0]], dtype=np.float32)
    d = np.array([[1, 0, 0], [0, 0, 0], [np.nan, 0, 1], [np.inf, 0, 0], [0, 0, 1], [1, 0, 0]], dtype=np.float32)
    r = _cast(occ, lab, o, d)
    assert (r["voxel"] == -1).all() and np.isinf(r["t"]).all() and (r["label"] == -1).all()
    assert (r["normal"] == 0).all()


def test_keep_mask():
    occ, lab = _grid([((4, 5, 6, 10, 6, 10), 1), ((8, 9, 6, 10, 6, 10), 2), ((12, 13, 6, 10, 6, 10), 200)])
    o, d = _net(-2, 8, 8), _ndir(1, 0, 0)
    assert _cast(occ, lab, o, d)["label"][0] == 1
    assert _cast(occ, lab, o, d, keep_words=OB.label_words([2]))["label"][0] == 2
    assert _cast(occ, lab, o, d, keep_words=OB.label_words([3]))["voxel"][0] == -1
    # a label outside [0, 127] is kept without a mask and never under one, whatever its bits
    assert _cast(occ, lab, _net(11, 8, 8), d)["label"][0] == 200
    assert _cast(occ, lab, _net(11, 8, 8), d, keep_words=[0xFFFFFFFF] * 4)["voxel"][0] == -1
    # NaN is never solid
    occ2 = occ.copy()
    occ2[4:6] = np.nan
    assert _cast(occ2, lab, o, d)["label"][0] == 2


def test_rotated_anisotropic_grid_hits_the_first_solid_voxel_along_the_ray():
    rng = np.random.default_rng(5)
    a = 0.7
    R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1.0]]) @ \
        np.array([[1, 0, 0], [0, np.cos(0.4), -np.sin(0.4)], [0, np.sin(0.4), np.cos(0.4)]])
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, (0.3, -0.2, 0.5)
    ext, dim = (1.9, 7.0, 4.0), 24
    occ = (rng.random((dim,) * 3) < 0.01).astype(np.float32) * rng.uniform(0.3, 1.0, (dim,) * 3).astype(np.float32)
    lab = rng.integers(0, 9, (dim,) * 3).astype(np.int16)
    n = 300
    inv, b = E.grid_index_map(T, ext, dim)
    centre = np.linalg.solve(inv, np.full(3, (dim - 1) / 2.0)) + b
    o = rng.uniform(-6, 6, (n, 3)).astype(np.float32)
    d = (centre + rng.uniform(-1.5, 1.5, (n, 3)) - o).astype(np.float32)
    r = G.cast(occ, lab, T, ext, o, d, 0.5, 30.0, level=0.45)
    assert (r["voxel"] >= 0).sum() > 30
    for q in range(n):
        u0 = inv @ (o[q].astype(np.float64) - b)
        w = inv @ d[q].astype(np.float64)
        t_end = float(r["t"][q]) if r["voxel"][q] >= 0 else 30.0
        ts = np.linspace(0.5, t_end, 400)[:-1]
        ts = ts[ts < t_end - 1e-6]
        u = u0[None] + ts[:, None] * w[None]
        inside = ((u >= -0.5) & (u <= dim - 0.5)).all(1)
        ii = np.clip(np.floor(u[inside] + 0.5), 0, dim - 1).astype(np.int64)
        assert not (occ[tuple(ii.T)] > np.float32(0.45)).any(), q          # nothing solid before the hit
        if r["voxel"][q] >= 0:
            qv = np.array(np.unravel_index(int(r["voxel"][q]), occ.shape))
            uh = u0 + float(r["t"][q]) * w
            assert (np.abs(uh - qv) <= 0.5 + 1e-5).all(), q                # the hit lies on the voxel's cube
            assert occ[tuple(qv)] > np.float32(0.45) and lab[tuple(qv)] == r["label"][q]
            assert abs(np.linalg.norm(r["normal"][q]) - 1.0) < 1e-12


def _cpu_grid(dim=4):
    return torch.zeros((dim,) * 3), torch.zeros((dim,) * 3, dtype=torch.int16)


@pytest.mark.parametrize("kw, msg", [
    (dict(near=2.0, far=1.0), "near"), (dict(near=float("nan")), "near"), (dict(far=float("inf")), "near"),
    (dict(level=float("nan")), "level"), (dict(keep=[1], remove=[2]), "at most one"), (dict(keep=[128]), "outside"),
    (dict(extents=(1.0, -1.0, 1.0)), "extents"), (dict(extents=(1.0, 1.0)), "extents"),
    (dict(scene_transform=np.diag([1.0, 1.0, -1.0, 1.0])), "determinant"), (dict(components={"label": []}), "components"),
])
def test_cast_grid_checks_its_arguments_before_device_work(kw, msg):
    occ, lab = _cpu_grid()
    args = dict(scene_transform=np.eye(4), near=0.0, far=1.0)
    args.update(kw)
    rays = torch.zeros(2, 3)
    with pytest.raises(ValueError, match=msg):
        OB.cast_grid(occ, lab, args.pop("scene_transform"), rays, rays, **args)


def test_cast_grid_needs_device_tensors():
    occ, lab = _cpu_grid()
    with pytest.raises(RuntimeError, match="CUDA"):
        OB.cast_grid(occ, lab, np.eye(4), torch.zeros(2, 3), torch.zeros(2, 3), 0.0, 1.0)


@pytest.mark.parametrize("kw, msg", [
    (dict(H=0), "H and W"), (dict(W=2.5), "H and W"), (dict(c2w=np.eye(3)), "c2w"), (dict(c2w=np.zeros((2, 2, 4))), "c2w"),
    (dict(lut=np.zeros((4, 3), dtype=np.int32)), "lut"), (dict(near=3.0, far=1.0), "near"),
])
def test_grid_view_checks_its_arguments_before_device_work(kw, msg):
    occ, lab = _cpu_grid()
    args = dict(H=4, W=4, K=np.eye(3), c2w=np.eye(4), near=0.0, far=1.0)
    args.update(kw)
    with pytest.raises(ValueError, match=msg):
        OB.grid_view(occ, lab, np.eye(4), **args)
