"""CPU: object selection -- the selection oracle (oracle/objects_oracle.py) against the fixture made from the original dm_nerf, object_mask, the RGBA PNG
writer and the command lines of tools/render_objects.py and tools/extract_mesh.py --per-object."""
import os
import struct
import sys
import zlib

import numpy as np
import pytest
import torch

from dmnerf_b200 import synth
from dmnerf_b200.objects import kept_labels, object_mask
from dmnerf_b200.tester import write_png
from oracle import dmnerf_oracle as O
from oracle import objects_oracle as OO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

MAPS = ("rgb_coarse", "depth_coarse", "acc_coarse", "ins_coarse", "weights_coarse", "rgb_fine", "depth_fine", "acc_fine",
        "ins_fine", "weights_fine", "z_vals_fine")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "objects.npz"))


@pytest.mark.parametrize("tag", ["study", "room0"])
def test_oracle_selection_matches_fixture(golden, tag):
    g = golden
    ins_num = int(g[tag + "_ins_num"])
    wc, wf = synth.make_weights(int(g["seed_coarse"]), ins_num), synth.make_weights(int(g["seed_fine"]), ins_num)
    ro, rd = torch.from_numpy(g[tag + "_rays_o"]), torch.from_numpy(g[tag + "_rays_d"])
    z = O.z_val_sample(ro.shape[0], float(g[tag + "_near"]), float(g[tag + "_far"]), 64)
    assert float(g[tag + "_min_gap"]) >= 1e-6
    for sel in ("keep", "remove", "empty"):
        p = "%s_%s_" % (tag, sel)
        keep = OO.keep_table(g[p + "mask"], ins_num + 1)
        with torch.no_grad():
            out = OO.render(ro, rd, O.to_torch(wc), O.to_torch(wf), z, keep)
        np.testing.assert_array_equal(OO.object_labels(out["raw_coarse"]).numpy(), g[p + "labels_coarse"])
        for k in MAPS:
            tol = 1e-5 if k.endswith("_coarse") else 2e-3       # the fine pass is ill-conditioned through sample_pdf
            np.testing.assert_allclose(out[k].numpy(), g[p + k], rtol=tol, atol=tol, err_msg="%s %s" % (p, k))
        if sel == "empty":
            for k in ("rgb_fine", "depth_fine", "acc_fine", "weights_fine", "rgb_coarse", "acc_coarse"):
                assert not g[p + k].any(), k
            assert (g[p + "ins_fine"] == 0.5).all()


def test_oracle_selection_keeps_raw_and_zeroes_only_density():
    g = np.random.default_rng(0)
    raw = torch.from_numpy(g.standard_normal((3, 7, 4 + 6)).astype(np.float32))
    keep = torch.tensor([True, False, True, False, False, True])
    sel = OO.select_objects(raw, keep)
    lab = OO.object_labels(raw)
    assert torch.equal(sel[..., :3], raw[..., :3]) and torch.equal(sel[..., 4:], raw[..., 4:])
    assert torch.equal(sel[..., 3], torch.where(keep[lab], raw[..., 3], torch.zeros_like(raw[..., 3])))


def test_object_mask_layout():
    assert object_mask(13, keep=[0, 5, 13]) == [(1 << 0) | (1 << 5) | (1 << 13), 0, 0, 0]
    assert object_mask(13, remove=[2]) == [((1 << 14) - 1) & ~(1 << 2), 0, 0, 0]
    assert object_mask(127, keep=[31, 32, 95, 127]) == [1 << 31, 1, 1 << 31, 1 << 31]
    assert object_mask(127, remove=[]) == [0xffffffff] * 4
    assert object_mask(93, keep=[]) == [0, 0, 0, 0]
    assert kept_labels(object_mask(59, remove=list(range(1, 60)))) == [0]
    assert kept_labels(object_mask(59, keep=(7, 40, 59))) == [7, 40, 59]
    assert object_mask(13, keep=np.array([3, 3], dtype=np.int64)) == [1 << 3, 0, 0, 0]


@pytest.mark.parametrize("kw", [dict(keep=[14]), dict(keep=[-1]), dict(remove=[20]), dict(keep=[1], remove=[2]), dict(),
                                dict(keep=[1.5]), dict(keep=[True])])
def test_object_mask_rejects(kw):
    with pytest.raises(ValueError):
        object_mask(13, **kw)


def _read_png(path):
    data = open(path, "rb").read()
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, chunks = 8, []
    while pos < len(data):
        n = struct.unpack(">I", data[pos:pos + 4])[0]
        tag, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        assert struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])[0] == zlib.crc32(tag + body) & 0xffffffff
        chunks.append((tag, body))
        pos += 12 + n
    assert [t for t, _ in chunks] == [b"IHDR", b"IDAT", b"IEND"]
    w, h, depth, ctype = struct.unpack(">IIBB", chunks[0][1][:10])
    ch = {0: 1, 2: 3, 6: 4}[ctype]
    raw = np.frombuffer(zlib.decompress(chunks[1][1]), np.uint8).reshape(h, 1 + w * ch)
    assert (raw[:, 0] == 0).all()
    return depth, ctype, raw[:, 1:].reshape(h, w, ch)


def test_write_png_rgba_round_trip(tmp_path):
    img = np.random.default_rng(1).integers(0, 256, (5, 11, 4), dtype=np.uint8)
    write_png(str(tmp_path / "a.png"), img)
    depth, ctype, back = _read_png(str(tmp_path / "a.png"))
    assert (depth, ctype) == (8, 6)
    np.testing.assert_array_equal(back, img)


def test_write_png_grey_and_rgb_bytes_unchanged(tmp_path):
    """Grey and RGB files are exactly the bytes the writer produced before RGBA was added (IHDR colour types 0 / 2)."""
    g = np.random.default_rng(2)
    for shape, ctype in (((6, 4), 0), ((6, 4, 3), 2)):
        img = g.integers(0, 256, shape, dtype=np.uint8)
        path = str(tmp_path / ("%d.png" % ctype))
        write_png(path, img)
        h, w = shape[:2]
        raw = np.concatenate([np.zeros((h, 1), np.uint8), img.reshape(h, -1)], 1).tobytes()

        def chunk(tag, data):
            return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xffffffff)

        expect = (b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, ctype, 0, 0, 0))
                  + chunk(b"IDAT", zlib.compress(raw, 6)) + chunk(b"IEND", b""))
        assert open(path, "rb").read() == expect
    with pytest.raises(ValueError):
        write_png(str(tmp_path / "bad.png"), np.zeros((2, 2, 2), np.uint8))


def test_render_objects_cli(tmp_path):
    import render_objects
    k = tmp_path / "K.npy"
    np.save(k, np.eye(3, dtype=np.float32))
    a = render_objects.parse(["ck.tar", "--pose", "p.npy", "--hwk", "48", "64", str(k), "--keep", "3", "5", "--out", "o"])
    assert (a.H, a.W, a.keep, a.remove, a.out) == (48, 64, [3, 5], None, "o")
    np.testing.assert_array_equal(a.K, np.eye(3))
    a = render_objects.parse(["ck.tar", "--pose", "p.npy", "--hwk", "4", "6", "1", "0", "2", "0", "-1", "3", "0", "0", "-1",
                              "--remove", "0", "--out", "o", "--near", "0.5"])
    assert a.remove == [0] and a.keep is None and a.near == 0.5 and a.K[1, 1] == -1 and a.K[2, 2] == -1
    for bad in (["ck.tar", "--pose", "p", "--hwk", "4", "6", "k.npy", "--out", "o"],                         # no selection
                ["ck.tar", "--pose", "p", "--hwk", "4", "6", "k.npy", "--keep", "1", "--remove", "2", "--out", "o"],
                ["ck.tar", "--pose", "p", "--hwk", "4", "6", "1", "2", "--keep", "1", "--out", "o"]):      # bad K
        with pytest.raises(SystemExit):
            render_objects.parse(bad)


def test_extract_mesh_cli():
    import extract_mesh
    a = extract_mesh.parse(["ck.tar", "T.npy", "--out", "o"])
    assert a.per_object is False and a.objects is None
    a = extract_mesh.parse(["ck.tar", "T.npy", "--out", "o", "--per-object", "--objects", "2", "7"])
    assert a.per_object is True and a.objects == [2, 7]
