"""GPU: labelled mesh extraction -- occupancy sweep, marching cubes, normals, clusters, cleanup, label rays, mesh_main."""
import json
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from dmnerf_b200 import mesh as M
from dmnerf_b200.testing import make_models
from oracle import dmnerf_oracle as O
from oracle import marching_cubes as MC

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "mesh_grid.npz"))


def _centered(n):
    x = np.arange(n, dtype=np.float64) - (n - 1) / 2.0
    return np.meshgrid(x, x, x, indexing="ij")


def sphere(n, r, c=(0.0, 0.0, 0.0)):
    X, Y, Z = _centered(n)
    return (r - np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2)).astype(np.float32)


def torus(n, R, r):
    X, Y, Z = _centered(n)
    return (r - np.sqrt((np.sqrt(X * X + Y * Y) - R) ** 2 + Z * Z)).astype(np.float32)


def noise(shape, seed):
    return np.random.default_rng(seed).random(shape).astype(np.float32)


def cases_of(g, level):
    ins = g > np.float32(level)
    nx, ny, nz = g.shape
    cube = np.zeros((nx - 1, ny - 1, nz - 1), dtype=np.int64)
    for c in range(8):
        a, b, d = c & 1, (c >> 1) & 1, (c >> 2) & 1
        cube |= ins[a:nx - 1 + a, b:ny - 1 + b, d:nz - 1 + d].astype(np.int64) << c
    return cube


def canon(tris):
    """Rotate every triangle so that its smallest index comes first (orientation kept)."""
    t = np.asarray(tris, dtype=np.int64)
    k = np.argmin(t, axis=1)
    return np.stack([t[np.arange(len(t)), (k + j) % 3] for j in range(3)], 1) if len(t) else t.reshape(0, 3)


def gpu_mc(g, level):
    v, t = M.marching_cubes(torch.from_numpy(g).to(DEV), level)
    return v.cpu().numpy(), t.cpu().numpy()


# ---- occupancy sweep -------------------------------------------------------------------------------------------------------

def test_grid_points_kernel_is_the_original_grid(golden):
    for tag in "ab":
        pts = M.grid_points(golden["transform_" + tag], int(golden["dim_" + tag]), golden["extents"], device=DEV)
        np.testing.assert_array_equal(pts.cpu().numpy(), golden["points_" + tag])
    part = M.grid_points(golden["transform_a"], 12, golden["extents"], begin=100, count=37, device=DEV)
    np.testing.assert_array_equal(part.cpu().numpy(), golden["points_a"][100:137])


@pytest.mark.parametrize("ins_num", [13, 93])
def test_occupancy_sweep_matches_the_oracle_network(golden, ins_num):
    _, nf, _, wf = make_models(101, 202, ins_num, DEV)
    T, dim, ext = golden["transform_a"], int(golden["dim_a"]), golden["extents"]
    near, far, n_imp = 4.0, 15.0, 128
    voxel = (far - near) / n_imp
    occ = M.occupancy_grid(nf, T, dim, ext, near, far, n_imp, slab=500, device=DEV)      # 1728 points: 3 full slabs + a ragged one
    assert occ.shape == (dim, dim, dim)
    pts = torch.from_numpy(golden["points_a"]).double()
    x = torch.cat([O.embed(pts, 10), O.embed(torch.zeros_like(pts), 4)], -1)
    sigma = O.mlp_forward(O.to_torch(wf, torch.float64), x)[:, 3]
    ref = (1.0 - torch.exp(-torch.relu(sigma) * voxel)).numpy()
    got = occ.reshape(-1).cpu().double().numpy()
    # the network's budget (1e-4 of the density channel's scale) carried through d occ / d sigma <= voxel
    tol = 1e-4 * voxel * float(sigma.abs().max()) + 2e-6
    assert np.abs(got - ref).max() <= tol, (np.abs(got - ref).max(), tol)
    assert 0.0 < ref.mean() < 1.0


# ---- marching cubes --------------------------------------------------------------------------------------------------------

FIELDS = {
    "sphere": lambda: (sphere(40, 15.2), 0.0),
    "torus": lambda: (torus(40, 11.0, 4.3), 0.0),
    "two_spheres": lambda: (np.maximum(sphere(40, 8.5, (-8.6, 0.3, 0.0)), sphere(40, 8.5, (8.6, -0.3, 0.2))), 0.0),
    "noise": lambda: (noise((24, 21, 19), 11), 0.45),
}


@pytest.mark.parametrize("name", sorted(FIELDS))
def test_marching_cubes_matches_the_table_free_oracle(name):
    g, level = FIELDS[name]()
    if name == "noise":
        assert len(np.unique(cases_of(g, level))) == 256
    v, t = gpu_mc(g, level)
    vo, to, _ = MC.marching_cubes(g, level)
    assert v.shape == vo.shape and t.shape == to.shape
    np.testing.assert_array_equal(v, vo)
    np.testing.assert_array_equal(canon(t), canon(to))


def test_marching_cubes_every_case_on_a_single_cell():
    rng = np.random.default_rng(2)
    for case in range(256):
        vals = rng.uniform(0.0, 0.44, 8).astype(np.float32)
        for c in range(8):
            if (case >> c) & 1:
                vals[c] = np.float32(rng.uniform(0.46, 1.0))
        g = np.zeros((2, 2, 2), dtype=np.float32)
        for c in range(8):
            g[c & 1, (c >> 1) & 1, (c >> 2) & 1] = vals[c]
        v, t = gpu_mc(g, 0.45)
        vo, to, _ = MC.marching_cubes(g, 0.45)
        np.testing.assert_array_equal(v, vo, err_msg="case %d" % case)
        np.testing.assert_array_equal(canon(t), canon(to), err_msg="case %d" % case)


def _boundary_plane(p, shape):
    return [(a, x) for a in range(3) for x in (0.0, shape[a] - 1.0) if p[a] == x]


def test_gpu_mesh_is_watertight_and_consistently_oriented():
    for name in ("sphere", "torus", "noise"):
        g, level = FIELDS[name]()
        v, t = gpu_mc(g, level)
        directed = np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]])
        _, n_dir = np.unique(directed, axis=0, return_counts=True)
        assert (n_dir == 1).all(), name                                # consistent orientation, manifold edges
        und, n_und = np.unique(np.sort(directed, 1), axis=0, return_counts=True)
        assert (n_und <= 2).all(), name
        for a, b in und[n_und == 1]:                                   # an open edge lies in a boundary plane of the grid
            assert set(_boundary_plane(v[a], g.shape)) & set(_boundary_plane(v[b], g.shape)), (name, v[a], v[b])
        if name != "noise":
            assert (n_und == 2).all(), name


def test_pipeline_is_bit_reproducible():
    g, level = FIELDS["noise"]()
    T = np.eye(4)
    runs = []
    for _ in range(2):
        v, t = M.marching_cubes(torch.from_numpy(g).to(DEV), level)
        vs = M.to_scene(v, T, 24)
        n = M.vertex_normals(vs, t)
        cl, sz = M.triangle_clusters(t, v.shape[0])
        runs.append([x.cpu().numpy() for x in (v, t, vs, n, cl, sz)])
    for a, b in zip(*runs):
        np.testing.assert_array_equal(a, b)


def test_nan_in_the_grid_is_rejected():
    g = sphere(16, 5.0)
    g[3, 4, 5] = np.nan
    with pytest.raises(RuntimeError, match="NaN"):
        M.marching_cubes(torch.from_numpy(g).to(DEV), 0.0)


# ---- normals, clusters, cleanup -------------------------------------------------------------------------------------------

def test_vertex_normals_match_numpy(golden):
    g, level = FIELDS["torus"]()
    v, t = M.marching_cubes(torch.from_numpy(g).to(DEV), level)
    vs = M.to_scene(v, golden["transform_a"], 40, golden["extents"])
    n = M.vertex_normals(vs, t).cpu().numpy()
    p, tt = vs.cpu().numpy().astype(np.float64), t.cpu().numpy()
    fn = np.cross(p[tt[:, 1]] - p[tt[:, 0]], p[tt[:, 2]] - p[tt[:, 0]])
    acc = np.zeros_like(p)
    for k in range(3):
        np.add.at(acc, tt[:, k], fn)
    ref = acc / np.linalg.norm(acc, axis=1, keepdims=True)
    assert np.abs(n - ref).max() < 1e-5
    # scene-space mapping: v / (dim - 1) in float32, then float64 (q - 0.5) * extents and the transform
    q = (v.cpu().numpy() / np.float32(39)).astype(np.float64)
    x = (q - 0.5) * 2.0 * (golden["extents"] / 2.0)
    T = golden["transform_a"]
    np.testing.assert_allclose(vs.cpu().numpy(), (x @ T[:3, :3].T + T[:3, 3]).astype(np.float32), rtol=0, atol=2e-6)


def _scipy_clusters(tris, nv):
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    nt = len(tris)
    e = np.concatenate([np.sort(tris[:, [0, 1]], 1), np.sort(tris[:, [1, 2]], 1), np.sort(tris[:, [2, 0]], 1)])
    key = e[:, 0].astype(np.int64) * nv + e[:, 1]
    tri = np.tile(np.arange(nt), 3)
    order = np.argsort(key, kind="stable")
    same = key[order][1:] == key[order][:-1]
    a, b = tri[order][:-1][same], tri[order][1:][same]
    n_comp, lab = connected_components(coo_matrix((np.ones(len(a)), (a, b)), shape=(nt, nt)), directed=False)
    first = np.full(n_comp, nt)
    np.minimum.at(first, lab, np.arange(nt))
    return first[lab], np.bincount(lab)[lab]


def blobs():
    g = sphere(48, 12.0, (-8.0, 0.0, 0.0))
    for c, r in (((14.0, 10.0, 9.0), 1.6), ((14.0, -11.0, -9.0), 2.3), ((15.0, 12.0, -12.0), 1.2), ((-12.0, 14.0, 14.0), 3.1)):
        g = np.maximum(g, sphere(48, r, c))
    return g


def test_clusters_match_scipy_connected_components():
    for g, level in (FIELDS["noise"](), (blobs(), 0.0)):
        v, t = M.marching_cubes(torch.from_numpy(g).to(DEV), level)
        cl, sz = M.triangle_clusters(t, v.shape[0])
        ref_cl, ref_sz = _scipy_clusters(t.cpu().numpy(), v.shape[0])
        np.testing.assert_array_equal(cl.cpu().numpy(), ref_cl)
        np.testing.assert_array_equal(sz.cpu().numpy(), ref_sz)


def test_cleanup_removes_small_clusters_and_keeps_order():
    v, t = M.marching_cubes(torch.from_numpy(blobs()).to(DEV), 0.0)
    n = M.vertex_normals(v, t)
    _, sz = _scipy_clusters(t.cpu().numpy(), v.shape[0])
    sizes = np.unique(sz)
    assert len(sizes) >= 4
    min_cluster = int(sizes[len(sizes) // 2])                   # some blobs above, some below
    cv, cn, ct = M.clean_mesh(v, n, t, min_cluster)
    tt = t.cpu().numpy()
    keep = sz >= min_cluster
    used = np.zeros(v.shape[0], bool)
    used[tt[keep].reshape(-1)] = True
    remap = np.cumsum(used) - 1
    np.testing.assert_array_equal(ct.cpu().numpy(), remap[tt[keep]])
    np.testing.assert_array_equal(cv.cpu().numpy(), v.cpu().numpy()[used])
    np.testing.assert_array_equal(cn.cpu().numpy(), n.cpu().numpy()[used])
    assert 0 < len(ct) < len(tt)


# ---- end to end --------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def e2e(golden):
    nc, nf, wc, wf = make_models(101, 202, 13, DEV, trained_like=True)
    T = golden["transform_a"]
    occ = M.occupancy_grid(nf, T, 64)
    lo, hi = float(occ.min()), float(occ.max())
    level = 0.45 if lo < 0.45 < hi else float(occ.float().quantile(0.5))
    out = M.extract_mesh(nf, nc, T, grid_dim=64, level=level, min_cluster=20, N_test=1000)
    return types.SimpleNamespace(nc=nc, nf=nf, wc=wc, wf=wf, T=T, level=level, out=out)


def test_extract_mesh_labels_are_the_renderers_argmax(e2e):
    from dmnerf_b200.render import render_rays
    out = e2e.out
    assert out["clean_vertices"].shape[0] > 0 and out["labels"].shape[0] == out["clean_vertices"].shape[0]
    # the label rays: mesh_generator.py:106-113 restated in numpy (float32, same operation order)
    v, n = out["clean_vertices"].cpu().numpy(), out["clean_normals"].cpu().numpy()
    rd = -n[:, [0, 2, 1]]
    rd[:, 1] *= -1
    vv = v[:, [0, 2, 1]].copy()
    vv[:, 1] *= -1
    ro = vv - (rd * np.float32(0.03)) * np.float32(4.0)
    np.testing.assert_array_equal(out["rays_d"].cpu().numpy(), rd)
    np.testing.assert_array_equal(out["rays_o"].cpu().numpy(), ro)
    from dmnerf_b200.helpers import z_val_sample
    z = z_val_sample(1, 0.01, 15, 64)[0].to(DEV)
    ref = render_rays(out["rays_o"], out["rays_d"], e2e.nc, e2e.nf, z, want_raw=False, want_coarse=False)
    assert torch.equal(out["labels"], torch.argmax(ref["ins_fine"], -1))


def test_extract_mesh_labels_agree_with_the_oracle_render(e2e):
    out = e2e.out
    n = out["rays_o"].shape[0]
    sel = np.random.default_rng(0).choice(n, min(512, n), replace=False)
    ro, rd = out["rays_o"][sel].cpu(), out["rays_d"][sel].cpu()
    ours = out["labels"][sel].cpu()
    ref = O.render(ro, rd, O.to_torch(e2e.wc), O.to_torch(e2e.wf), O.z_val_sample(len(sel), 0.01, 15, 64))
    twin = O.render(ro.double(), rd.double(), O.to_torch(e2e.wc, torch.float64), O.to_torch(e2e.wf, torch.float64),
                    O.z_val_sample(len(sel), 0.01, 15, 64, dtype=torch.float64))
    agree = float((ours == ref["ins_fine"].argmax(-1)).float().mean())
    agree_twin = float((twin["ins_fine"].argmax(-1) == ref["ins_fine"].argmax(-1)).float().mean())
    assert agree >= agree_twin - 0.05, (agree, agree_twin)


def test_mesh_main_writes_both_files(e2e, tmp_path):
    from dmnerf_b200.embedder import get_embedder
    args = types.SimpleNamespace(near=4.0, far=15.0, N_samples=64, N_importance=128, N_test=2048, expname="study",
                                 datadir="./data/dmsr/study")
    rgbs = np.random.default_rng(1).integers(0, 256, (20, 3))
    color_dict = {str(k): k for k in range(20)}
    ins_map = {str(k): (k + 1) % 14 for k in range(13)}
    out = M.mesh_main(get_embedder(10)[0], get_embedder(4)[0], e2e.nc, e2e.nf, args, None, rgbs, str(tmp_path), ins_map,
                      scene_transform=e2e.T, color_dict=color_dict, grid_dim=64, level=e2e.level, min_cluster=20)
    a, b = M.read_ply(tmp_path / "study.ply"), M.read_ply(tmp_path / "color_study.ply")
    np.testing.assert_array_equal(a["vertices"], out["vertices"].cpu().numpy())
    np.testing.assert_array_equal(a["faces"], out["triangles"].cpu().numpy())
    np.testing.assert_array_equal(b["vertices"], out["clean_vertices"].cpu().numpy())
    np.testing.assert_array_equal(b["faces"], out["clean_triangles"].cpu().numpy())
    want = M.label_colors(out["labels"], rgbs, color_dict, ins_map)[:, ::-1]
    np.testing.assert_array_equal(b["colors"], want)


def test_extract_mesh_command_line_on_a_checkpoint(tmp_path):
    nc, nf, _, _ = make_models(7, 8, 13, "cpu", trained_like=True)
    torch.save({"network_coarse_state_dict": nc.state_dict(), "network_fine_state_dict": nf.state_dict()}, tmp_path / "ck.tar")
    np.save(tmp_path / "T.npy", np.eye(4))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "extract_mesh.py"), str(tmp_path / "ck.tar"), str(tmp_path / "T.npy"),
                        "--out", str(tmp_path / "o"), "--name", "m", "--grid-dim", "48", "--min-cluster", "1"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    info = json.loads(r.stdout.strip().splitlines()[-1])
    a, b = M.read_ply(tmp_path / "o" / "m.ply"), M.read_ply(tmp_path / "o" / "color_m.ply")
    assert (len(a["vertices"]), len(a["faces"])) == (info["vertices"], info["triangles"])
    assert (len(b["vertices"]), len(b["faces"])) == (info["clean_vertices"], info["clean_triangles"])
    assert b["colors"] is not None and len(b["colors"]) == len(b["vertices"])
