"""CPU: deforming objects (DESIGN.md, "Deforming objects") -- the pull inverts the forward map, the destination box holds the
deformed object, the identity table is the rigid move bit for bit, a constant quarter turn is the rigid quarter turn, an integer
shear of a pole is per-layer shifting, a twisted and tapered piece keeps its height range; the rejections of the Python layer, the
tool and the library, and the new prototypes and struct."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from dmnerf_b200 import _lib
from dmnerf_b200 import objects as OB
from oracle import deform_oracle as DO
from oracle import edit_sweep_oracle as E
from oracle import group_oracle as GO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T, DIM, EXT, LEVEL = np.eye(4), 17, (4.0, 4.0, 4.0), 0.45     # grid points and 0.25 steps exact in fp32
UP, FWD = (0.0, 0.0, 1.0), (1.0, 0.0, 0.0)                  # network z is index axis 1, network x index axis 0


def _random_table(rng, K):
    th = np.cumsum(rng.uniform(-0.5, 0.5, K))
    sc = rng.uniform(0.6, 1.4, K)
    A = np.stack([np.stack([np.cos(th) * sc, -np.sin(th) * sc], -1), np.stack([np.sin(th) * sc, np.cos(th) * sc], -1)], 1)
    A[:, 0, 1] += rng.uniform(-0.2, 0.2, K)                      # a shear: not a similarity
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    q = q * np.sign(np.linalg.det(q))
    return OB.Deformation(rng.uniform(-0.5, 0.5, 3), q[:, 2], q[:, 0], rng.uniform(-1, 0), rng.uniform(0.05, 0.3), A,
                          rng.uniform(-0.3, 0.3, (K, 2)))


def _pole_scene():
    occ = np.zeros((DIM,) * 3, dtype=np.float32)
    labels = np.zeros((DIM,) * 3, dtype=np.int16)
    occ[4, 3:12, 8], labels[4, 3:12, 8] = 0.9, 1
    return occ, labels


def test_the_pull_inverts_the_forward_map():
    rng = np.random.default_rng(0)
    for K in (2, 5, 33, 64):
        d = _random_table(rng, K)
        x = rng.uniform(-2, 2, (2000, 3))
        back, _ = DO.pull(d, DO.forward(d, x))
        assert np.abs(back - x).max() <= 1e-12, K


def test_the_forward_images_of_the_source_box_lie_in_the_destination_box():
    rng = np.random.default_rng(1)
    inv, b = E.grid_index_map(T, EXT, DIM)
    A = np.linalg.inv(inv)
    for trial in range(20):
        d = _random_table(rng, int(rng.integers(2, 12)))
        lo = rng.integers(0, DIM - 6, 3)
        box = [int(v) for a in range(3) for v in (lo[a], lo[a] + rng.integers(0, 6))]
        trans = np.eye(4)
        trans[:3, 3] = rng.uniform(-0.5, 0.5, 3)
        mv = {"trans": trans, "box": box, "deform": d}
        dlo, dhi = DO.destination_box(mv, T, EXT, DIM)
        u = np.stack([rng.uniform(box[2 * a] - 0.5, box[2 * a + 1] + 0.5, 4000) for a in range(3)], -1)
        y = DO.forward(d, u @ A.T + b[None, :])                     # the source point where it lands before the move
        p = (y - trans[:3, 3][None, :]) @ np.linalg.inv(trans[:3, :3]).T
        idx = (p - b[None, :]) @ inv.T
        inside = np.all((idx >= -0.5) & (idx <= DIM - 0.5), axis=1)
        q = np.rint(idx[inside])
        assert ((q >= dlo) & (q <= dhi)).all(), trial


def test_the_identity_table_takes_the_rigid_decisions_bit_for_bit():
    rng = np.random.default_rng(2)
    occ = rng.uniform(0, 1, (DIM,) * 3).astype(np.float32)
    labels = rng.integers(0, 4, (DIM,) * 3).astype(np.int16)
    ident = OB.Deformation((0, 0, 0), UP, FWD, -2.0, 0.5, [np.eye(2)] * 9, np.zeros((9, 2)))
    inv, b = E.grid_index_map(T, EXT, DIM)
    pts = E.sweep_points(T, EXT, DIM)
    trans = np.eye(4)
    trans[:3, :3] = [[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]]
    trans[:3, 3] = (0.37, -0.11, 0.2)
    for rigid in ({"label": 1, "trans": trans, "box": (2, 14, 0, 16, 3, 12)},
                  {"label": 2, "trans": np.eye(4), "box": (0, 16, 0, 16, 0, 16), "copy": True, "group": [2, 3]}):
        deformed = dict(rigid, deform=ident)
        assert np.array_equal(DO.targets(deformed, pts), E.targets(trans if rigid["label"] == 1 else np.eye(4), pts))
        want = GO.grid_edit(occ, labels, occ, labels, T, EXT, [dict(rigid, group=rigid.get("group", [rigid["label"]]))], LEVEL)
        got = DO.grid_edit(occ, labels, occ, labels, T, EXT, [deformed], LEVEL)
        for w, g in zip(want, got):
            assert np.array_equal(w, g)
        assert np.array_equal(DO.move_overlap(occ, labels, T, EXT, [deformed], LEVEL)[0],
                              GO.move_overlap(occ, labels, T, EXT, [dict(rigid, group=rigid.get("group", [rigid["label"]]))],
                                              LEVEL)[0])
    # the view direction: J^-1 of the identity is the identity
    w = rng.normal(size=(100, 3))
    _, st = DO.pull(ident, rng.uniform(-2, 2, (100, 3)))
    assert np.array_equal(DO.direction(ident, st, w), w)


def test_a_constant_quarter_turn_about_a_grid_point_is_the_rigid_quarter_turn():
    rng = np.random.default_rng(3)
    occ = rng.uniform(0, 1, (DIM,) * 3).astype(np.float32)
    labels = rng.integers(0, 3, (DIM,) * 3).astype(np.int16)
    c = np.array([0.25, -0.5, 0.75])
    Aq = np.array([[0.0, -1.0], [1.0, 0.0]])
    turn = OB.Deformation(c, UP, FWD, -1.0, 0.25, [Aq] * 4, np.zeros((4, 2)))
    R = np.array([[0.0, 1.0, 0.0], [-1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])   # x = c + R (y - c): the pull of the turn
    rigid = np.eye(4)
    rigid[:3, :3], rigid[:3, 3] = R, c - R @ c
    pts = E.sweep_points(T, EXT, DIM)
    assert np.array_equal(DO.targets({"trans": np.eye(4), "deform": turn}, pts), E.targets(rigid[:3], pts))
    box = (0, 16, 0, 16, 0, 16)
    got = DO.grid_edit(occ, labels, occ, labels, T, EXT, [{"label": 1, "trans": np.eye(4), "box": box, "deform": turn}], LEVEL)
    want = GO.grid_edit(occ, labels, occ, labels, T, EXT, [{"label": 1, "trans": rigid, "box": box, "group": [1]}], LEVEL)
    for w, g in zip(want, got):
        assert np.array_equal(w, g)


def test_an_integer_shear_of_a_pole_is_per_layer_shifting():
    occ, labels = _pole_scene()
    layers = np.arange(3, 12)
    z = -2.0 + 0.25 * layers                                      # network z of index j
    K = len(layers)
    shear = OB.Deformation((0, 0, 0), UP, FWD, float(z[0]), 0.25, [np.eye(2)] * K, np.stack([0.25 * np.arange(K), np.zeros(K)], -1))
    box = (2, 6, 1, 13, 6, 10)
    o, l, landed, _ = DO.grid_edit(occ, labels, occ, labels, T, EXT, [{"label": 1, "trans": np.eye(4), "box": box,
                                                                         "deform": shear}], LEVEL)
    want = np.zeros((DIM,) * 3, dtype=bool)
    for k, j in enumerate(layers):
        want[:, j, :] = np.roll(occ[:, j, :] > LEVEL, k, axis=0)
    assert np.array_equal(o > LEVEL, want) and (l[want] == 1).all() and landed[0] == K


def test_a_twisted_and_tapered_piece_keeps_its_height_range():
    occ = np.zeros((DIM,) * 3, dtype=np.float32)
    labels = np.zeros((DIM,) * 3, dtype=np.int16)
    occ[5:12, 3:13, 5:12], labels[5:12, 3:13, 5:12] = 0.9, 2
    d = OB.deformation((0.0, 0.0, 0.0), UP, -1.25, 1.25, 9, twist=lambda s: 70.0 * s, taper=lambda s: 1.0 - 0.4 * s)
    o, l, _, _ = DO.grid_edit(occ, labels, occ, labels, T, EXT, [{"label": 2, "trans": np.eye(4), "box": (3, 13, 1, 15, 3, 13),
                                                                    "deform": d}], LEVEL)
    solid = (o > LEVEL) & (l == 2)
    js = np.nonzero(solid.any(axis=(0, 2)))[0]
    assert js.min() == 3 and js.max() == 12
    assert solid.sum() != ((occ > LEVEL) & (labels == 2)).sum() or not np.array_equal(solid, (occ > LEVEL) & (labels == 2))


def test_the_builder_frames_and_profiles():
    d = OB.deformation((1.0, 2.0, 3.0), (0, 0, 2.0), 0.0, 1.0, 5, twist=[0, 10, 20, 30, 40], bend=lambda s: s, bend_dir=(1, 1, 5))
    np.testing.assert_allclose(d.frame[:3], [2 ** -0.5, 2 ** -0.5, 0], atol=1e-15)
    np.testing.assert_allclose(d.frame[6:9], [0, 0, 1])
    assert d.dh == 0.25 and d.knots.shape == (5, 6)
    np.testing.assert_allclose(d.knots[:, 4], np.linspace(0, 1, 5))
    th = np.radians(40.0)
    np.testing.assert_allclose(d.knots[-1, :4], [np.cos(th), -np.sin(th), np.sin(th), np.cos(th)])
    assert OB.move_deformations(None, 2) is None and OB.move_deformations([None, None], 2) is None
    assert OB.move_deformations([d, None], 2)[0] is d
    for bad in ([d], d, "x"):
        with pytest.raises(ValueError, match="deformations must be"):
            OB.move_deformations(bad, 2)


# ---- rejections: Python, the tool and the library give one message ----------------------------------------------------------------

def _bad_tables():
    I = np.eye(2)
    ok = dict(centre=(0, 0, 0), up=UP, forward=FWD, h0=0.0, dh=1.0, A=[I, I], t=np.zeros((2, 2)))
    return [
        (dict(ok, A=[I], t=np.zeros((1, 2))), "n_knots 1 is not 0 and outside [2, 64]"),
        (dict(ok, A=[I] * 65, t=np.zeros((65, 2))), "n_knots 65 is not 0 and outside [2, 64]"),
        (dict(ok, h0=np.inf), "a value is not finite"),
        (dict(ok, t=[[0, 0], [np.nan, 0]]), "a value is not finite"),
        (dict(ok, dh=0.0), "dh 0 must be > 0"),
        (dict(ok, up=(0, 0, 1.001)), "the frame is not orthonormal and right-handed"),
        (dict(ok, forward=(1, 1e-4, 0)), "the frame is not orthonormal and right-handed"),
        (dict(ok, A=[I, -I]), "det A(h) <= 0 on knot interval 0"),
        (dict(ok, A=[I, I, np.diag([1.0, -1.0])], t=np.zeros((3, 2))), "det A(h) <= 0 on knot interval 1"),
    ]


def _abi(kw):
    up, fwd = np.asarray(kw["up"], dtype=np.float64), np.asarray(kw["forward"], dtype=np.float64)
    A, t = np.asarray(kw["A"], dtype=np.float64), np.asarray(kw["t"], dtype=np.float64)
    knots = np.concatenate([A.reshape(-1, 4), t], 1)
    held = (C.c_double * knots.size)(*knots.reshape(-1).tolist())
    d = _lib.Deformation()
    d.n_knots, d.h0, d.dh, d.knots = knots.shape[0], float(kw["h0"]), float(kw["dh"]), C.cast(held, C.POINTER(C.c_double))
    d.frame[:] = np.concatenate([fwd, np.cross(up, fwd), up, np.asarray(kw["centre"], dtype=np.float64)]).tolist()
    return (_lib.Deformation * 2)(_lib.Deformation(), d), held


def test_python_and_the_library_reject_a_table_with_the_same_message():
    lib = _lib.load()
    calls = {
        "mesh_occupancy_edit_deformed": lambda d: lib.dmnerf_mesh_occupancy_edit_deformed(None, 0, None, None, 17, 0.1, 0.45, 0, None, None,
                                                                                         None, d, 2, None, None, None, None),
        "grid_edit_deformed": lambda d: lib.dmnerf_grid_edit_deformed(None, None, None, 17, 0.45, None, None, None, None, None, d, 2,
                                                                      None, None, None, None, None),
        "move_overlap_deformed": lambda d: lib.dmnerf_move_overlap_deformed(None, None, None, 17, 0.45, None, None, None, None, None, d,
                                                                            2, None, None, None, None),
    }
    moves = _lib.RenderMoves()
    moves.n_moves = 2
    calls["render_moved_deformed"] = lambda d: lib.dmnerf_render_moved_deformed(None, None, 1, 64, 128, 0, 0, C.byref(moves), None,
                                                                                None, d, None, None)
    for kw, msg in _bad_tables():
        with pytest.raises(ValueError) as e:
            OB.Deformation(**kw)
        assert str(e.value) == "deformation: " + msg
        arr, held = _abi(kw)
        for who, call in calls.items():
            assert call(arr) != 0
            assert lib.dmnerf_last_error().decode() == "%s: move 1: deformation: %s" % (who, msg), who
    bad = _lib.Deformation()
    bad.n_knots = 3
    assert calls["grid_edit_deformed"]((_lib.Deformation * 2)(_lib.Deformation(), bad)) != 0
    assert lib.dmnerf_last_error().decode() == "grid_edit_deformed: move 1: deformation: the knot table is NULL"
    # an all-rigid array passes the deformation checks and fails on what comes next
    assert calls["grid_edit_deformed"]((_lib.Deformation * 2)()) != 0
    assert "deformation" not in lib.dmnerf_last_error().decode()


def test_the_tool_takes_the_deformation_flags_and_rejects_as_the_library(capsys):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import move_objects
    base = ["ck.tar", "--pose", "p.npy", "--hwk", "4", "4"] + ["1"] * 9 + ["--transform", "t.npy", "--out", "o"]
    mv = ["--move-label", "1", "--mode", "translation", "--render", "samples"]
    a = move_objects.parse(base + mv + ["--twist", "30", "--up", "0", "0", "1", "--mesh", "--check"])
    assert a.deformed and a.twist == 30.0 and a.knots == 33 and a.mesh and a.check
    a = move_objects.parse(base + mv + ["--bend", "0.1", "--bend-dir", "1", "0", "0", "--taper", "0.8", "--up", "0", "0", "1",
                                        "--knots", "9"])
    assert a.bend == 0.1 and a.bend_dir == [1.0, 0.0, 0.0] and a.taper == 0.8 and a.knots == 9
    place = ["--move-label", "1", "--place-at", "0", "0", "0", "--down", "0", "-1", "0", "--render", "samples"]
    for extra, msg in ((["--move-label", "1", "--mode", "translation", "--twist", "3", "--up", "0", "0", "1"], "--render samples"),
                       (place + ["--twist", "3", "--up", "0", "0", "1"], "--place-at"),
                       (mv + ["--until-contact", "--twist", "3", "--up", "0", "0", "1"], "--until-contact"),
                       (mv + ["--twist", "3"], "--up"),
                       (mv + ["--bend", "1", "--up", "0", "0", "1"], "--bend-dir"),
                       (mv + ["--up", "0", "0", "1"], "need --twist"),
                       (mv + ["--twist", "3", "--up", "0", "0", "1", "--knots", "1"], "deformation: n_knots 1 is not 0 and outside [2, 64]"),
                       (mv + ["--taper", "-1", "--up", "0", "0", "1"], "deformation: taper must be > 0")):
        with pytest.raises(SystemExit):
            move_objects.parse(base + extra)
        assert msg in capsys.readouterr().err, msg
    for kw, msg in ((dict(knots=1, twist=[0]), "deformation: n_knots 1 is not 0 and outside [2, 64]"),
                    (dict(taper=lambda s: -1.0), "deformation: taper must be > 0")):
        with pytest.raises(ValueError) as e:
            OB.deformation((0, 0, 0), UP, 0.0, 1.0, **kw)
        assert str(e.value) == msg


def test_the_deformed_entry_points_are_the_group_ones_with_a_deformation_argument(tmp_path):
    P = _lib.PROTOTYPES
    defs = C.POINTER(_lib.Deformation)
    for name, at in (("dmnerf_mesh_occupancy_edit", 11), ("dmnerf_grid_edit", 10), ("dmnerf_render_moved", 10),
                     ("dmnerf_move_overlap", 10)):
        base, new = P[name + "_groups"], P[name + "_deformed"]
        assert new[0] is base[0] and new[1][at] is defs and new[1][:at] + new[1][at + 1:] == base[1], name
    hdr = open(os.path.join(ROOT, "include", "dmnerf_b200.h")).read()
    for name in ("dmnerf_mesh_occupancy_edit", "dmnerf_grid_edit", "dmnerf_render_moved", "dmnerf_move_overlap"):
        proto = re.search(r"DMNERF_API int %s_deformed\(([^;]*)\);" % name, hdr).group(1)
        group = re.search(r"DMNERF_API int %s_groups\(([^;]*)\);" % name, hdr).group(1)
        strip = lambda s: [re.sub(r"/\*.*?\*/", "", x).split()[-1].strip("*") for x in s.split(",")]
        args, gargs = strip(proto), strip(group)
        assert [x for x in args if x != "deformations_host"] == gargs, name
    src = tmp_path / "layout.c"
    fields = [f[0] for f in _lib.Deformation._fields_]
    src.write_text("#include <stddef.h>\n#include <stdio.h>\n#include \"dmnerf_b200.h\"\nint main(void) {\n"
                   '  printf("sizeof %%zu\\n", sizeof(dmnerf_deformation));\n%s\n  return 0;\n}\n'
                   % "\n".join('  printf("%s %%zu\\n", offsetof(dmnerf_deformation, %s));' % (f, f) for f in fields))
    exe = str(tmp_path / "layout")
    subprocess.run(["cc", "-std=c11", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe], check=True)
    got = dict(line.split() for line in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["sizeof"]) == C.sizeof(_lib.Deformation)
    assert all(int(got[f]) == getattr(_lib.Deformation, f).offset for f in fields)
