"""GPU: object selection in the fused render kernel, the stage kernels, the frame driver and the occupancy sweep; one mesh per
object; the two command-line tools."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from dmnerf_b200 import _lib, synth
from dmnerf_b200 import mesh as M
from dmnerf_b200.engine import get_context
from dmnerf_b200.manipulator import exchanger
from dmnerf_b200.objects import meshes_from_labelled_grid, object_mask, object_meshes, occupancy_objects
from dmnerf_b200.render import composite, render_frame, render_rays
from dmnerf_b200.testing import format_parity_table, make_models, parity_table
from oracle import dmnerf_oracle as O
from oracle import objects_oracle as OO

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
MAPS = ("rgb_coarse", "depth_coarse", "acc_coarse", "ins_coarse", "rgb_fine", "depth_fine", "acc_fine", "ins_fine")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "objects.npz"))


def cu(a):
    return torch.as_tensor(np.asarray(a)).to(DEV).contiguous()


def _rays(name, n, first=0):
    wl = synth.workload(name)
    sel = np.linspace(first, wl["H"] * wl["W"] - 1, n).astype(np.int64)
    return wl, cu(wl["rays_o"][sel]), cu(wl["rays_d"][sel])


def _z(wl, n=1):
    return O.z_val_sample(n, wl["near"], wl["far"], 64)[0].to(DEV)


def _equal(a, b, keys):
    for k in keys:
        assert torch.equal(a[k], b[k]), k


# ------------------------------------------------------------------------------------------ nothing changes without a selection
@pytest.mark.parametrize("name,ins_num,impl", [
    pytest.param("dmsr_study", 13, _lib.IMPL_AUTO, id="dmsr_study"),
    pytest.param("replica_room0_93", 93, _lib.IMPL_AUTO, id="replica_room0_93"),
    # the fp16 preview network's selected kernel (render_objects_f16_kernel) at 2, 14 and 128 label channels
    pytest.param("dmsr_study", 1, _lib.IMPL_UMMA_F16, id="dmsr_study-f16-ins1"),
    pytest.param("dmsr_study", 13, _lib.IMPL_UMMA_F16, id="dmsr_study-f16-ins13"),
    pytest.param("dmsr_study", 127, _lib.IMPL_UMMA_F16, id="dmsr_study-f16-ins127")])
def test_keep_all_is_bit_identical(name, ins_num, impl):
    """A selection that keeps every label gives the unselected maps bit for bit: fused kernel (impl), stage kernels (SIMT),
    frame driver (impl)."""
    wl, ro, rd = _rays(name, 1024)
    nc, nf, _, _ = make_models(101, 202, ins_num, DEV)
    everything = list(range(ins_num + 1))
    with torch.no_grad():
        fused = render_rays(ro, rd, nc, nf, _z(wl), want_raw=False, want_samples=True, impl=impl)
        fused_sel = render_rays(ro, rd, nc, nf, _z(wl), want_raw=False, want_samples=True, keep_objects=everything, impl=impl)
        _equal(fused, fused_sel, fused.keys())
        simt = render_rays(ro, rd, nc, nf, _z(wl), impl=_lib.IMPL_SIMT)
        simt_sel = render_rays(ro, rd, nc, nf, _z(wl), impl=_lib.IMPL_SIMT, keep_objects=everything)
        _equal(simt, simt_sel, simt.keys())
        K, c2w = wl["K"], wl["c2w"]
        fr = render_frame(wl["H"], wl["W"], K, c2w, wl["near"], wl["far"], nc, nf, pixel_range=(100000, 8192), device=DEV,
                          impl=impl)
        fr_sel = render_frame(wl["H"], wl["W"], K, c2w, wl["near"], wl["far"], nc, nf, pixel_range=(100000, 8192), device=DEV,
                              keep_objects=everything, impl=impl)
        _equal(fr, fr_sel, fr.keys())
    get_context(DEV).sync_check()


# ------------------------------------------------------------------------------------------ against the original and the oracle
def test_teacher_forced_selected_composite(golden):
    g = golden
    p = "study_remove_"
    raw = g[p + "raw_fine"]
    n = raw.shape[0]
    z, rd = g[p + "z_vals_fine"][:n], g["study_rays_d"][:n]
    kept = [k for k in range(14) if (int(g[p + "mask"][k >> 5]) >> (k & 31)) & 1]
    with torch.no_grad():
        rgb, w, depth, ins, acc = composite(cu(raw), cu(z), cu(rd), keep_objects=kept)
        ref = O.composite(OO.select_objects(torch.from_numpy(raw), OO.keep_table(g[p + "mask"], 14)), torch.from_numpy(z),
                          torch.from_numpy(rd))
    for got, want, floor in ((rgb, ref[0], 1e-2), (w, ref[1], 1e-3), (depth, ref[2], 1e-1), (ins, ref[3], 1e-2), (acc, ref[4], 1e-2)):
        err = np.max(np.abs(got.cpu().numpy() - want.numpy()) / np.maximum(np.abs(want.numpy()), floor))
        assert err <= 1e-4, err
    # the fixture's own maps (the original dm_nerf, teacher-forced on the same raw)
    np.testing.assert_allclose(w.cpu().numpy(), g[p + "weights_fine"][:n], rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("tag", ["study", "room0"])
def test_simt_end_to_end_vs_original(golden, tag):
    g = golden
    ins_num = int(g[tag + "_ins_num"])
    nc, nf, wc, wf = make_models(int(g["seed_coarse"]), int(g["seed_fine"]), ins_num, DEV)
    ro, rd = cu(g[tag + "_rays_o"]), cu(g[tag + "_rays_d"])
    n = ro.shape[0]
    z = O.z_val_sample(n, float(g[tag + "_near"]), float(g[tag + "_far"]), 64)[0].to(DEV)
    for sel in ("keep", "remove", "empty"):
        p = "%s_%s_" % (tag, sel)
        kept = [k for k in range(ins_num + 1) if (int(g[p + "mask"][k >> 5]) >> (k & 31)) & 1]
        keep = OO.keep_table(g[p + "mask"], ins_num + 1)
        with torch.no_grad():
            out = render_rays(ro, rd, nc, nf, z, impl=_lib.IMPL_SIMT, keep_objects=kept)
            twin = OO.render(ro.cpu().double(), rd.cpu().double(), O.to_torch(wc, torch.float64), O.to_torch(wf, torch.float64),
                            O.z_val_sample(n, float(g[tag + "_near"]), float(g[tag + "_far"]), 64, dtype=torch.float64), keep)
        np.testing.assert_array_equal(OO.object_labels(out["raw_coarse"].cpu()).numpy(), g[p + "labels_coarse"])
        np.testing.assert_allclose(out["rgb_coarse"].cpu().numpy(), g[p + "rgb_coarse"], rtol=1e-4, atol=1e-5)
        for k, floor in (("z_vals_fine", 1e-3), ("rgb_fine", 1e-4), ("depth_fine", 1e-3), ("ins_fine", 1e-4)):
            ref = g[p + k]
            dev_twin = float(np.abs(twin[k].float().numpy() - ref).max())
            dev_ours = float(np.abs(out[k].cpu().numpy() - ref).max())
            assert dev_ours <= 10.0 * dev_twin + floor, (p, k, dev_ours, dev_twin)


@pytest.mark.parametrize("sel", ["keep", "remove"])
def test_fused_vs_live_oracle(golden, sel):
    """The fused kernel with a selection against the live oracle on 2048 rays, the oracle's fp64 twin as the yard-stick: the twin
    also moves where the fine pass is ill-conditioned and where a near-tied label flips.  No ray is excluded."""
    top = int(golden["study_top"])
    wl, ro, rd = _rays("dmsr_study", 2048)
    ins_num = wl["ins_num"]
    nc, nf, wc, wf = make_models(101, 202, ins_num, DEV)
    kept = [top] if sel == "keep" else [k for k in range(ins_num + 1) if k != top]
    keep = torch.zeros(ins_num + 1, dtype=torch.bool)
    keep[kept] = True
    n = ro.shape[0]
    z = O.z_val_sample(n, wl["near"], wl["far"], 64)
    with torch.no_grad():
        ours = render_rays(ro, rd, nc, nf, z[0].to(DEV), want_raw=False, want_samples=False, keep_objects=kept)
        ref = OO.render(ro.cpu(), rd.cpu(), O.to_torch(wc), O.to_torch(wf), z, keep)
        twin = OO.render(ro.cpu().double(), rd.cpu().double(), O.to_torch(wc, torch.float64), O.to_torch(wf, torch.float64),
                        O.z_val_sample(n, wl["near"], wl["far"], 64, dtype=torch.float64), keep)
        # label flips: the tensor-core network's labels against the fp32 oracle's on the oracle's own samples
        from dmnerf_b200.autograd import mlp_forward_rays
        flips = []
        for net, zk, rk in ((nc, "z_vals_coarse", "raw_coarse"), (nf, "z_vals_fine", "raw_fine")):
            raw = mlp_forward_rays(net, ro, rd, ref[zk].to(DEV).contiguous())
            flips.append(float((OO.object_labels(raw.cpu()) != OO.object_labels(ref[rk])).double().mean()))
    table = parity_table(ours, twin, ref)
    print("\n" + format_parity_table("dmsr_study %s {%d} (2048 rays)" % (sel, top), table))
    print("label flips, tensor-core vs fp32 logits: coarse %.2e, fine %.2e of samples" % tuple(flips))
    assert max(flips) <= 1e-2
    for k, row in table.items():
        o, t = row["ours"], row["twin"]
        assert o["n"] == n
        assert o["frac_within"] >= t["frac_within"] - 0.03, (k, o, t)
        assert o["median"] <= 2.0 * t["median"] + 1e-6, (k, o, t)
        assert o["p99"] <= 2.0 * t["p99"] + 1e-4, (k, o, t)


# ------------------------------------------------------------------------------------------ semantics
def test_removed_object_carries_no_weight():
    wl, ro, rd = _rays("dmsr_study", 512)
    ins_num = wl["ins_num"]
    nc, nf, _, _ = make_models(101, 202, ins_num, DEV)
    with torch.no_grad():
        base = render_rays(ro, rd, nc, nf, _z(wl), impl=_lib.IMPL_SIMT)
        lab = OO.object_labels(base["raw_fine"].cpu())
        mass = torch.zeros(ins_num + 1, dtype=torch.float64).index_add_(0, lab.reshape(-1), base["weights_fine"].cpu().double().reshape(-1))
        k = int(mass.argmax())
        out = render_rays(ro, rd, nc, nf, _z(wl), impl=_lib.IMPL_SIMT, keep_objects=[j for j in range(ins_num + 1) if j != k])
    for raw_key, w_key in (("raw_coarse", "weights_coarse"), ("raw_fine", "weights_fine")):
        hit = OO.object_labels(out[raw_key].cpu()) == k
        assert bool(hit.any()), raw_key
        assert bool((out[w_key].cpu()[hit] == 0).all()), w_key
    assert float(out["acc_fine"].sum()) < float(base["acc_fine"].sum())


@pytest.mark.parametrize("impl", [_lib.IMPL_AUTO, _lib.IMPL_SIMT])
def test_empty_selection_and_reproducibility(impl):
    wl, ro, rd = _rays("replica_room0", 600)
    nc, nf, _, _ = make_models(101, 202, wl["ins_num"], DEV)
    want_raw = impl == _lib.IMPL_SIMT
    with torch.no_grad():
        e = render_rays(ro, rd, nc, nf, _z(wl), impl=impl, want_raw=want_raw, keep_objects=[])
        a = render_rays(ro, rd, nc, nf, _z(wl), impl=impl, want_raw=want_raw, keep_objects=[0, 3, 17])
        b = render_rays(ro, rd, nc, nf, _z(wl), impl=impl, want_raw=want_raw, keep_objects=[0, 3, 17])
    for s in ("coarse", "fine"):
        for k in ("rgb_", "depth_", "acc_"):
            assert bool((e[k + s] == 0).all()), k + s
        assert bool((e["ins_" + s] == 0.5).all())
    _equal(a, b, a.keys())


# ------------------------------------------------------------------------------------------ rejections
def test_selection_is_rejected_outside_the_labels_at_every_entry_point():
    wl, ro, rd = _rays("dmsr_study", 64)
    nc, nf, _, _ = make_models(101, 202, 13, DEV)
    with torch.no_grad():
        with pytest.raises(ValueError):
            render_rays(ro, rd, nc, nf, _z(wl), keep_objects=[14])
        with pytest.raises(ValueError):
            render_frame(48, 64, wl["K"], wl["c2w"], 4.0, 15.0, nc, nf, device=DEV, keep_objects=[-1])
    with pytest.raises(RuntimeError, match="inference-only"):
        render_rays(ro, rd, nc, nf, _z(wl), keep_objects=[1])                   # parameters require grad, grad enabled
    big, _, _, _ = make_models(303, 404, 59, DEV)
    with torch.no_grad(), pytest.raises(RuntimeError):
        render_rays(ro, rd, nc, big, _z(wl), keep_objects=[1])
    # the C ABI itself: a bit at or above ins_num + 1 is rejected by every entry point that takes a selection, naming the label
    ctx = get_context(DEV)
    ctx.bind(0, nc); ctx.bind(1, nf)
    n, st, lib = ro.shape[0], ctx.stream(), ctx.lib
    bad = (C.c_uint32 * 4)(1 << 14, 0, 0, 0)
    edit = _lib.Edit(keep=C.cast(bad, C.POINTER(C.c_uint32)))
    z, out = _z(wl), torch.empty(n, 3, device=DEV)                        # every buffer a native call reads stays referenced
    io = _lib.RenderIO(rays_o=ro.data_ptr(), rays_d=rd.data_ptr(), z_coarse=z.data_ptr(), rgb_fine=out.data_ptr(),
                       edit=C.pointer(edit))
    ro_h, rd_h, z_h, out_h = ro.cpu(), rd.cpu(), z.cpu(), torch.empty(n, 3)
    io_h = _lib.RenderIO(rays_o=ro_h.data_ptr(), rays_d=rd_h.data_ptr(), z_coarse=z_h.data_ptr(), rgb_fine=out_h.data_ptr(),
                         edit=C.pointer(edit))
    Kf, Cf = _lib.camera(wl["K"], wl["c2w"])
    raw, z_rows = torch.rand(n, 64, 18, device=DEV), z.expand(n, 64).contiguous()
    rgb, w, depth, ins, acc = (torch.empty(n, 3, device=DEV), torch.empty(n, 64, device=DEV), torch.empty(n, device=DEV),
                               torch.empty(n, 13, device=DEV), torch.empty(n, device=DEV))
    comp = (raw.data_ptr(), z_rows.data_ptr(), rd.data_ptr(), n, 64, 18, 0)
    comp_out = (rgb.data_ptr(), w.data_ptr(), depth.data_ptr(), ins.data_ptr(), acc.data_ptr(), st)
    eye = (C.c_double * 16)(*np.eye(4).reshape(-1)); ext = (C.c_double * 3)(1.9, 7.0, 7.0)
    occ, lab = torch.empty(8, 8, 8, device=DEV), torch.empty(8, 8, 8, device=DEV, dtype=torch.int16)
    calls = {
        "render_forward": lambda: lib.dmnerf_render_forward(ctx.handle, io, n, 64, 128, 0, 0, st),
        "render_forward_host": lambda: lib.dmnerf_render_forward_host(ctx.handle, io_h, n, 64, 128, 0, 0, st),
        "render_frame_host": lambda: lib.dmnerf_render_frame_host(ctx.handle, Kf, Cf, 48, 64, 4.0, 15.0, 0, n, 64, 128, 0, 0,
                                                                  C.byref(io_h), st),
        "composite": lambda: lib.dmnerf_composite(*comp, bad, *comp_out),
        "mesh_occupancy": lambda: lib.dmnerf_mesh_occupancy(ctx.handle, 1, eye, ext, 8, 0.1, 0, bad, occ.data_ptr(), lab.data_ptr(), st),
    }
    for name, call in calls.items():
        assert call() != 0, name
        err = lib.dmnerf_last_error()
        assert name.encode() in err and b"keeps label 14, outside [0, 13]" in err, (name, err)
    # without an edit (io->edit NULL, or an edit whose members are all NULL) and with a NULL mask: the unselected result, bit
    # for bit
    with torch.no_grad():
        ref = render_rays(ro, rd, nc, nf, z, want_raw=False, want_samples=False)
    for e in (None, C.pointer(_lib.Edit())):
        io.edit = io_h.edit = e
        _lib.check(lib.dmnerf_render_forward(ctx.handle, io, n, 64, 128, 0, 0, st), "dmnerf_render_forward")
        assert torch.equal(out, ref["rgb_fine"])
        _lib.check(lib.dmnerf_render_forward_host(ctx.handle, io_h, n, 64, 128, 0, 0, st), "dmnerf_render_forward_host")
        assert torch.equal(out_h, ref["rgb_fine"].cpu())
    everything = _lib.keep_mask(object_mask(13, remove=[]))
    _lib.check(lib.dmnerf_composite(*comp, None, *comp_out), "dmnerf_composite")
    plain = [t.clone() for t in (rgb, w, depth, ins, acc)]
    _lib.check(lib.dmnerf_composite(*comp, everything, *comp_out), "dmnerf_composite")
    assert all(torch.equal(a, b) for a, b in zip(plain, (rgb, w, depth, ins, acc)))
    _lib.check(lib.dmnerf_mesh_occupancy(ctx.handle, 1, eye, ext, 8, 0.1, 0, None, occ.data_ptr(), None, st), "dmnerf_mesh_occupancy")
    plain = occ.clone()
    _lib.check(lib.dmnerf_mesh_occupancy(ctx.handle, 1, eye, ext, 8, 0.1, 0, everything, occ.data_ptr(), lab.data_ptr(), st),
               "dmnerf_mesh_occupancy")
    assert torch.equal(occ, plain)
    # the unselected sweep does not write labels: asking it for them is an error, not a silently untouched buffer
    assert lib.dmnerf_mesh_occupancy(ctx.handle, 1, eye, ext, 8, 0.1, 0, None, occ.data_ptr(), lab.data_ptr(), st) != 0
    assert b"labels" in lib.dmnerf_last_error()
    ctx.sync_check()


# ------------------------------------------------------------------------------------------ meshes
def _transform():
    T = np.eye(4)
    T[:3, 3] = (0.1, -0.2, 0.3)
    return T


def test_selected_sweep_and_labels():
    nc, nf, _, _ = make_models(101, 202, 13, DEV)
    T, dim = _transform(), 40
    with torch.no_grad():
        occ_full = M.occupancy_grid(nf, T, dim, device=DEV)
        pts = M.grid_points(T, dim, device=DEV)
        from dmnerf_b200.autograd import mlp_forward_points
        raw = mlp_forward_points(nf, pts, torch.zeros_like(pts)).reshape(dim ** 3, 1, -1).contiguous()
        # argmax_sigmoid through the exchanger with a label no sample has: no edit, ori_label = the per-sample label
        acc = torch.zeros(dim ** 3, 14, device=DEV)
        _, _, label, _ = exchanger(raw.clone(), [raw], acc, [acc], [-1])
        label = label.reshape(dim, dim, dim)
        present = torch.unique(label).cpu().tolist()
        for kept in ([present[0]], [k for k in range(14) if k != present[0]], list(range(14)), []):
            occ, lab = occupancy_objects(nf, T, object_mask(13, keep=kept), dim, device=DEV)
            keep = torch.zeros(14, dtype=torch.bool, device=DEV)
            keep[kept] = True
            assert torch.equal(lab.long(), label)
            assert torch.equal(occ, torch.where(keep[label], occ_full, torch.zeros_like(occ_full)))
        # the same label as torch's argmax wherever the top two sigmoids are clearly apart
        s = torch.sigmoid(raw[:, 0, 4:].double())
        top = torch.topk(s, 2, -1).values
        clear = (top[:, 0] - top[:, 1]) > 1e-6
        assert torch.equal(label.reshape(-1)[clear], torch.argmax(s, -1)[clear])


def test_object_meshes_equal_masked_marching_cubes():
    nc, nf, _, _ = make_models(101, 202, 13, DEV)
    T, dim = _transform(), 48
    with torch.no_grad():
        occ, lab = occupancy_objects(nf, T, object_mask(13, remove=[13]), dim, device=DEV)
        sample = occ.flatten().float()
        level = float(sample.kthvalue(int(0.97 * sample.numel())).values)
        objs = [k for k in torch.unique(lab).cpu().tolist() if k != 13][:3]
        meshes = object_meshes(nf, nc, T, objects=objs, grid_dim=dim, level=level, min_cluster=0)
        assert sorted(meshes) == sorted(objs)
        for k in objs:
            v, t = M.marching_cubes(torch.where(lab == k, occ, torch.zeros_like(occ)), level)
            assert torch.equal(meshes[k]["triangles"], t)
            assert torch.equal(meshes[k]["vertices"], M.to_scene(v, T, dim))
        default = object_meshes(nf, nc, T, grid_dim=dim, level=level, min_cluster=0)
        assert 13 not in default and set(objs) <= set(default)


def _edge_use(tris):
    t = tris.cpu().numpy().astype(np.int64)
    e = np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]])
    e.sort(1)
    _, counts = np.unique(e, axis=0, return_counts=True)
    return counts


def test_per_object_meshes_are_closed():
    """Two touching boxes on an analytic labelled grid: label 1 inside, label 2 against it and clipped by the grid boundary."""
    n = 24
    occ = torch.zeros(n, n, n, device=DEV)
    lab = torch.zeros(n, n, n, device=DEV, dtype=torch.int16)
    occ[5:12, 6:14, 4:15] = 1.0
    lab[5:12, 6:14, 4:15] = 1
    occ[12:, 3:20, 2:18] = 1.0                    # touches box 1 at x = 12 and reaches the x = n - 1 face
    lab[12:, 3:20, 2:18] = 2
    meshes = meshes_from_labelled_grid(occ, lab, np.eye(4), [1, 2], level=0.45, min_cluster=0)
    inner = _edge_use(meshes[1]["triangles"])
    assert inner.size and (inner == 2).all()
    outer = _edge_use(meshes[2]["triangles"])
    assert (outer == 1).any()                     # open where the grid boundary clips it, as a whole-scene mesh is
    assert (outer <= 2).all()


# ------------------------------------------------------------------------------------------ the tools, end to end
def _checkpoint(tmp_path, ins_num=13):
    nc, nf, _, _ = make_models(7, 8, ins_num, "cpu")
    path = str(tmp_path / "ck.tar")
    torch.save({"network_coarse_state_dict": nc.state_dict(), "network_fine_state_dict": nf.state_dict()}, path)
    return path


def test_render_objects_tool(tmp_path):
    from dmnerf_b200.tester import write_png     # noqa: F401  (the files are PNG from the package's writer)
    ck = _checkpoint(tmp_path)
    wl = synth.workload("dmsr_study")
    H, W = 48, 64
    K = synth.dmsr_intrinsics(H, W)
    np.save(str(tmp_path / "pose.npy"), np.stack([wl["c2w"], synth.pose_spherical(40.0, -65.0, 7.0)]))
    out = str(tmp_path / "out")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "render_objects.py"), ck, "--pose", str(tmp_path / "pose.npy"),
                        "--hwk", str(H), str(W)] + [repr(float(v)) for v in K.reshape(-1)] + ["--remove", "13", "--out", out],
                       capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["frames"] == 2
    assert sorted(os.listdir(out)) == ["000.png", "001.png", "instance_000.png", "instance_001.png"]
    data = open(os.path.join(out, "000.png"), "rb").read()
    assert data[25] == 6                          # IHDR colour type: RGBA


def test_extract_mesh_per_object_tool(tmp_path):
    ck = _checkpoint(tmp_path)
    np.save(str(tmp_path / "T.npy"), np.eye(4))
    out = str(tmp_path / "mesh")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "extract_mesh.py"), ck, str(tmp_path / "T.npy"), "--out", out,
                        "--grid-dim", "48", "--min-cluster", "1", "--per-object"], capture_output=True, text=True, cwd=ROOT,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    objs = [f for f in res["files"] if "_obj" in f]
    assert res["files"][:2] == ["mesh.ply", "color_mesh.ply"] and objs
    for f in res["files"]:
        M.read_ply(os.path.join(out, f))
