"""Generate tests/golden/mani_eval.npz from the UNMODIFIED original loops manipulator_eval / manipulator_demo
(networks/manipulator.py:208-491), run on the CPU at a tiny size.

The original module imports packages that are not needed to run its loops on the CPU; they are replaced for the import:
  lpips            a model that returns NaN (the LPIPS column is NaN on both sides),
  skimage.metrics  oracle/metrics.py (PSNR / SSIM restated from scikit-image 0.18.3),
  imageio / cv2    imwrite captures the arrays instead of writing files,
  open3d / matplotlib  empty modules, so that tools/visualizer.py's real render_label2img / render_gt_label2img load.
torch.rand (sample_pdf's draw) is fed a pre-drawn uniform stream: rows of a torch.Generator seeded with `useed_<case>`, taken in
the order the original asks for them.  ./data/color_dict.json is a synthetic table in a temporary directory.

Cases: eval (2 frames, one moved object, gt perturbed from the original's own edited render so that matches and misses both
occur), demo_rigid (2 moved objects, 2 views), demo_deform (5 deformed objects, one per deformation function, 2 views).
Stored: the inputs, the uniform stream's seed and checksum, the original's per-frame maps (recorded by wrapping the module's
`manipulator` global), its fp64 deformation offsets, every captured image, matching_log.json and test_results.txt.

    DMNERF_REFERENCE_ROOT=<checkout of the original> python oracle/make_golden_mani_eval.py"""
import io
import json
import os
import sys
import tempfile
import types
from contextlib import redirect_stdout

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ["DMNERF_REFERENCE_ROOT"]
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)

from oracle import metrics as OM                                            # noqa: E402
from oracle import dmnerf_oracle as O                                       # noqa: E402

CAPTURED = {}


def _standins():
    class _NanLpips:
        def to(self, device):
            return self

        def __call__(self, a, b):
            return torch.tensor(float("nan"))

    lp = types.ModuleType("lpips")
    lp.LPIPS = lambda net="vgg": _NanLpips()
    sk = types.ModuleType("skimage")
    skm = types.ModuleType("skimage.metrics")
    skm.peak_signal_noise_ratio = lambda a, b, data_range=1: OM.psnr(a, b)
    skm.structural_similarity = lambda a, b, multichannel=True, data_range=1: OM.ssim(a, b)
    sk.metrics = skm

    def imwrite(path, img):
        CAPTURED[path] = np.array(img, copy=True)
        return True

    imageio, cv2 = types.ModuleType("imageio"), types.ModuleType("cv2")
    imageio.imwrite = cv2.imwrite = imwrite
    mpl, plt = types.ModuleType("matplotlib"), types.ModuleType("matplotlib.pyplot")
    mpl.pyplot = plt
    for name, m in (("lpips", lp), ("skimage", sk), ("skimage.metrics", skm), ("imageio", imageio), ("cv2", cv2),
                    ("open3d", types.ModuleType("open3d")), ("matplotlib", mpl), ("matplotlib.pyplot", plt)):
        sys.modules[name] = m


_standins()
import networks.manipulator as RM                                          # noqa: E402
from networks.dm_nerf import DM_NeRF as RefNet, get_embedder as ref_get_embedder   # noqa: E402
from dmnerf_b200 import synth                                               # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
INS_NUM, H, W, S, NI, N_TEST = 13, 24, 32, 16, 32, 300


class UniformStream:
    """torch.rand stand-in: successive rows of one pre-drawn [rows, NI] uniform table."""

    def __init__(self, u):
        self.u, self.pos = u, 0

    def __call__(self, *size, **kw):
        shape = list(size[0]) if len(size) == 1 and isinstance(size[0], (list, tuple, torch.Size)) else list(size)
        assert shape[-1] == NI, shape
        rows = int(np.prod(shape[:-1]))
        out = self.u[self.pos:self.pos + rows].reshape(shape)
        assert out.shape[0] == rows, "uniform stream exhausted"
        self.pos += rows
        return out


def uniforms(seed, rows):
    return torch.rand(rows, NI, generator=torch.Generator().manual_seed(seed))


def ref_net(weights_np):
    net = RefNet(8, 256, 63, 27, [4], INS_NUM)
    net.load_state_dict({k: torch.from_numpy(v) for k, v in weights_np.items()})
    return net.eval()


def weights(rays_o, rays_d, z):
    """Synthetic networks whose instance heads read the feature's deviation from its mean over the frame's coarse samples, so
    that the labels vary across the image (a random head on synthetic features gives one label everywhere)."""
    wc, wf = synth.make_weights(31, INS_NUM), synth.make_weights(32, INS_NUM)
    for seed, w in ((5, wc), (6, wf)):
        p = O.to_torch(w)
        x, _ = O._net_inputs(rays_o, rays_d, rays_d / torch.norm(rays_d, dim=-1, keepdim=True), z)
        h = x[..., :63]
        for i in range(O.N_TRUNK):
            h = torch.relu(O._lin(p, "mlps.%d" % i, h))
            if i in O.SKIPS:
                h = torch.cat([h, x[..., :63]], -1)
        f = torch.relu(O._lin(p, "ins_feature_linears.0", O._lin(p, "ins_feature_linear", h))).double().numpy()
        g = np.random.Generator(np.random.PCG64(seed)).standard_normal((INS_NUM + 1, f.shape[1])) * 10 / np.sqrt(f.shape[1])
        head = g / (f.std(0) + 1e-6)
        w["ins_linear.weight"] = head.astype(np.float32)
        w["ins_linear.bias"] = (-head @ f.mean(0)).astype(np.float32)
    return wc, wf


def rot_z(ang, shift):
    c, s = np.cos(ang), np.sin(ang)
    return np.array([[c, -s, 0, shift[0]], [s, c, 0, shift[1]], [0, 0, 1, shift[2]], [0, 0, 0, 1]], np.float32)


class Recorder:
    """Wraps the module's `manipulator` global: keeps every chunk's (final rgb, final ins)."""

    def __init__(self):
        self.inner, self.chunks = RM.manipulator, []

    def __call__(self, *a):
        out = self.inner(*a)
        self.chunks.append((out[0].clone(), out[1].clone()))
        return out

    def frames(self):
        per = -(-H * W // N_TEST)
        assert len(self.chunks) % per == 0
        rgb = [torch.cat([c[0] for c in self.chunks[f:f + per]]) for f in range(0, len(self.chunks), per)]
        ins = [torch.cat([c[1] for c in self.chunks[f:f + per]]) for f in range(0, len(self.chunks), per)]
        return torch.stack(rgb).numpy(), torch.stack(ins).numpy()


def run(fn, stream, *a, **k):
    """fn(*a, **k) with torch.rand fed from `stream` and the module's manipulator recorded; returns (recorder, stdout)."""
    rec = Recorder()
    real_rand = torch.rand
    RM.manipulator, torch.rand = rec, stream
    buf = io.StringIO()
    try:
        with torch.no_grad(), redirect_stdout(buf):
            fn(*a, **k)
    finally:
        RM.manipulator, torch.rand = rec.inner, real_rand
    assert stream.pos == stream.u.shape[0], (stream.pos, stream.u.shape)
    return rec, buf.getvalue()


def captured(prefix, save_dir):
    out = {}
    for path, img in sorted(CAPTURED.items()):
        assert os.path.dirname(path) == save_dir, path
        out["img_%s_%s" % (prefix, os.path.basename(path)[:-4])] = img
    CAPTURED.clear()
    return out


def main():
    wl = synth.workload("dmsr_study")
    K = np.array(wl["K"], dtype=np.float32).copy()
    K[:2] *= np.float32(W / wl["W"])                             # the workload's field of view at H x W
    K[0, 2], K[1, 2] = W / 2, H / 2
    c2w = np.asarray(wl["c2w"], dtype=np.float32)
    poses = np.stack([c2w + _shift(c2w, f) for f in range(2)])
    o, d = O.get_rays_k(H, W, K, torch.from_numpy(c2w))
    with torch.no_grad():
        wc, wf = weights(o.reshape(-1, 3), d.reshape(-1, 3), O.z_val_sample(H * W, wl["near"], wl["far"], S))
    nc, nf = ref_net(wc), ref_net(wf)
    pe, ve = ref_get_embedder(10)[0], ref_get_embedder(4)[0]
    rng = np.random.default_rng(23)
    ins_rgbs = rng.integers(0, 256, (40, 3))
    color_dict = {str(i): i for i in range(0, 30)}
    near, far = float(wl["near"]), float(wl["far"])
    store = dict(ins_num=INS_NUM, H=H, W=W, n_samples=S, n_importance=NI, n_test=N_TEST, near=near, far=far, K=K, poses=poses,
                 ins_rgbs=ins_rgbs, color_dict=json.dumps(color_dict), seed_c=31, seed_f=32, ins_w_c=wc["ins_linear.weight"],
                 ins_b_c=wc["ins_linear.bias"], ins_w_f=wf["ins_linear.weight"], ins_b_f=wf["ins_linear.bias"])
    base = dict(datadir="./data/dmsr/study", device=torch.device("cpu"), ins_num=INS_NUM, N_test=N_TEST, N_samples=S,
                N_importance=NI, near=near, far=far)
    tmp = tempfile.mkdtemp()
    os.makedirs(os.path.join(tmp, "data"))
    with open(os.path.join(tmp, "data", "color_dict.json"), "w") as fh:
        json.dump({"dmsr": {"study": color_dict}}, fh)
    os.chdir(tmp)

    # ---- eval: one move; the gt is the original's own edited render, perturbed -------------------------------------------
    trans = rot_z(0.3, (0.4, -0.2, 0.1))
    trans_dicts = {"transformations": [{"mode": "translation", "transformation": trans.tolist()}]}
    rows = 2 * (2 + 1) * H * W
    u = uniforms(101, rows)
    args = types.SimpleNamespace(target_label=2, **base)
    # pre-pass: the same loop body (manipulator.py:233-273) without the metrics, on the same uniforms
    rec = Recorder()
    stream = UniformStream(u)
    real_rand = torch.rand
    torch.rand = stream
    try:
        with torch.no_grad():
            args.target_labels = [args.target_label]
            for pose in torch.from_numpy(poses):
                o, d = RM.get_rays_k(H, W, K, pose)
                to, td = RM.get_rays_k(H, W, K, torch.from_numpy(trans) @ pose)
                o, d, to, td = o.reshape(-1, 3), d.reshape(-1, 3), to.reshape(-1, 3), td.reshape(-1, 3)
                for s in range(0, H * W, N_TEST):
                    e = min(s + N_TEST, H * W)
                    rec(pe, ve, nc, nf, torch.stack([o[s:e], d[s:e]]), torch.stack([to[s:e], td[s:e]])[None], args)
    finally:
        torch.rand = real_rand
    pre_rgb, pre_ins = rec.frames()
    gt_rgbs, gt_labels = [], []
    for f in range(2):
        lab = pre_ins[f][:, :-1].argmax(-1).reshape(H, W)
        ids, counts = np.unique(lab, return_counts=True)
        for small in ids[np.argsort(counts)][:max(0, len(ids) - 10)]:        # at most 10 + 1 gt objects for ins_num 13
            lab[lab == small] = ids[np.argmax(counts)]
        lab = lab + 3                                                            # gt ids differ from predicted labels
        lab[2 + f:9 + f, 4:13] = 20 + f                                          # an object nothing predicts: a miss
        gt_labels.append(lab)
        noisy = pre_rgb[f].reshape(H, W, 3) + 0.03 * rng.standard_normal((H, W, 3))
        gt_rgbs.append(np.clip(noisy, 0, 1).astype(np.float32))
    gt_labels = np.stack(gt_labels).astype(np.int8)
    gt_rgbs = np.stack(gt_rgbs)
    save = os.path.join(tmp, "eval")
    rec, log = run(RM.manipulator_eval, UniformStream(u), pe, ve, nc, nf, torch.from_numpy(poses), (H, W, K), trans_dicts, save,
                   ins_rgbs, args, gt_rgbs=torch.from_numpy(gt_rgbs), gt_labels=torch.from_numpy(gt_labels))
    rgb, ins = rec.frames()
    assert np.array_equal(rgb, pre_rgb) and np.array_equal(ins, pre_ins)
    sd = os.path.join(save, "translation")
    store.update(eval_trans=trans, eval_target_label=2, eval_useed=101, eval_usum=float(u.double().sum()), eval_rgb=rgb,
                 eval_ins=ins, eval_gt_rgbs=gt_rgbs, eval_gt_labels=gt_labels, eval_stdout=log,
                 eval_matching_log=open(os.path.join(sd, "matching_log.json")).read(),
                 eval_test_results=open(os.path.join(sd, "test_results.txt")).read(), **captured("eval", sd))
    print(log)

    # ---- demo: rigid (2 objects) and deform (5 objects, one per function), 2 views --------------------------------------
    view_poses = torch.from_numpy(poses)
    ins_map = {str(l): l + 3 for l in range(0, INS_NUM + 1, 2)}
    store["demo_ins_map"] = json.dumps(ins_map)
    cases = {
        "rigid": [{"obj_name": "chair", "tar_id": 2, "mani_mode": "rigid"}, {"obj_name": "lamp", "tar_id": 7, "mani_mode": "rigid"}],
        "deform": [{"obj_name": "o%d" % j, "tar_id": t, "mani_mode": "deform", "deform_func": fn}
                   for j, (t, fn) in enumerate(zip((1, 2, 4, 7, 11), ("sin", "ex", "linear", "abs_linear", "ln")))],
    }
    objs_trans = {"chair": [{"transformation": rot_z(0.2 * v, (0.3, 0.1 * v, 0.0)).tolist()} for v in range(2)],
                  "lamp": [{"transformation": rot_z(-0.25, (-0.2 * v, 0.2, 0.15)).tolist()} for v in range(2)]}
    store["demo_objs_trans"] = json.dumps(objs_trans)
    for name, objs in cases.items():
        seed = 202 if name == "rigid" else 303
        u = uniforms(seed, 2 * (2 + len(objs)) * H * W)
        args = types.SimpleNamespace(mani_type=name, **base)
        offsets = []
        real_from_numpy = torch.from_numpy

        def from_numpy(a):
            if a.dtype == np.float64 and a.size == H * W:
                offsets.append(a.copy())
            return real_from_numpy(a)

        torch.from_numpy = from_numpy
        try:
            rec, log = run(RM.manipulator_demo, UniformStream(u), pe, ve, nc, nf, poses, (H, W, K), objs_trans, tmp, ins_rgbs,
                           objs, view_poses, ins_map, args)
        finally:
            torch.from_numpy = real_from_numpy
        rgb, ins = rec.frames()
        sd = os.path.join(tmp, name)
        store.update({"demo_%s_objs" % name: json.dumps(objs), "demo_%s_useed" % name: seed,
                      "demo_%s_usum" % name: float(u.double().sum()), "demo_%s_rgb" % name: rgb, "demo_%s_ins" % name: ins},
                     **captured("demo_" + name, sd))
        if name == "deform":
            assert len(offsets) == 2 * len(objs)
            per_row = np.stack([o.reshape(H, W)[:, 0] for o in offsets]).reshape(2, len(objs), H)   # [view, function, H]
            assert all(np.array_equal(o.reshape(H, W), np.repeat(o.reshape(H, W)[:, :1], W, 1)) for o in offsets)
            store["demo_deform_offsets"] = per_row
        print(log)
    np.savez_compressed(os.path.join(OUT, "mani_eval.npz"), **store)
    print("written tests/golden/mani_eval.npz", os.path.getsize(os.path.join(OUT, "mani_eval.npz")) // 1024, "KB")


def _shift(c2w, f):
    p = np.zeros_like(c2w)
    p[:3, 3] = np.float32(0.05 * f)
    return p


if __name__ == "__main__":
    main()
